"""The graph index on the device against tests/_graph_oracle.py: the build bit for bit from the device's own k-NN
lists, the search bit for bit against the replay on small-integer tables, full coverage, batch invariance, a recall
floor, persistence, the Milvus shim and the workspace contract."""
from __future__ import annotations

import ctypes

import numpy as np
import pytest
import torch

from recnn_b200 import _lib
from recnn_b200.data import ItemIndex, ItemSets, MilvusConnection
from recnn_b200.utils.metrics import recall_at_k
from tests import _exact_retrieval as X
from tests import _graph_oracle as G
from tests.test_workspace_bounds_serving_gpu import check_windows, _ptr, set_args, set_table

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
L = _lib.lib()
METRICS = ["L2", "IP", "COS"]


def _np(t):
    return t.detach().cpu().numpy()


def _selves(n):
    return ItemSets(torch.arange(n, device=DEV), torch.arange(n + 1, device=DEV))


def _mixture(n, dim, n_blobs, seed):
    rng = np.random.default_rng(seed)
    centers = rng.standard_normal((n_blobs, dim))
    lab = rng.integers(0, n_blobs, n)
    return (centers[lab] + rng.standard_normal((n, dim))).astype(np.float32)


# ---------------------------------------------------------------------------------------------------- build
@pytest.mark.parametrize("d,D", [(16, 32), (32, 64), (64, 64)])
@pytest.mark.parametrize("dim", [13, 64, 132])
@pytest.mark.parametrize("metric", METRICS)
def test_graph_matches_oracle(metric, dim, d, D):
    n = 1200
    table = torch.randn(n, dim, device=DEV, generator=torch.Generator(device=DEV).manual_seed(dim + d))
    index = ItemIndex(table, metric)
    knn = index.knn_lists(D)
    want = ItemIndex(table, metric).search(table, D, exclude=_selves(n), exclude_rows=torch.arange(n, device=DEV)).ids
    assert torch.equal(knn, want)
    index.build_graph(graph_degree=d, intermediate_degree=D)
    g = _np(index.graph)
    np.testing.assert_array_equal(g, G.build(_np(knn), d))
    assert g.dtype == np.int32 and g.shape == (n, d)
    np.testing.assert_array_equal(_np(index.graph_entry), _np(torch.randperm(n, generator=torch.Generator()
                                                                               .manual_seed(0))[:512]))


@pytest.mark.parametrize("metric", METRICS)
def test_ivf_knn_stage_searches_short_rows_again(metric):
    n, D = 400, 32
    table = torch.randn(n, 16, device=DEV, generator=torch.Generator(device=DEV).manual_seed(1))
    index = ItemIndex(table, metric)
    got = index.knn_lists(D, knn_nlist=16, knn_nprobe=1)
    ivf = ItemIndex(table, metric).build_ivf(16)
    rows = torch.arange(n, device=DEV)
    want = ivf.search(table, D, search_param={"nprobe": 1}, exclude=_selves(n), exclude_rows=rows).ids
    short = (want < 0).any(1)
    assert int(short.sum()) > 0                                  # lists of 25 items on average: some row finds fewer than 32
    exact = ItemIndex(table, metric).search(table, D, exclude=_selves(n), exclude_rows=rows).ids
    want[short] = exact[short]
    assert torch.equal(got, want)
    index.build_graph(16, D, knn_nlist=16, knn_nprobe=1)
    np.testing.assert_array_equal(_np(index.graph), G.build(_np(want), 16))


def test_build_is_bit_reproducible_and_replaces_ivf():
    table = torch.randn(3000, 48, device=DEV, generator=torch.Generator(device=DEV).manual_seed(2))
    a = ItemIndex(table, "L2").build_ivf(16)
    a.build_graph(32, 48)
    assert a.ivf is None and a.graph is not None
    b = ItemIndex(table, "L2").build_graph(32, 48)
    assert torch.equal(a.graph, b.graph) and torch.equal(a.graph_entry, b.graph_entry)
    a.build_ivf(16)
    assert a.graph is None and a.ivf is not None


def test_build_refuses_bad_arguments():
    table = torch.randn(100, 8, device=DEV)
    for kw in [dict(graph_degree=24), dict(graph_degree=32, intermediate_degree=16),
               dict(graph_degree=64, intermediate_degree=96)]:
        with pytest.raises(ValueError):
            ItemIndex(table, "L2").build_graph(**kw)
    with pytest.raises(ValueError):
        ItemIndex(table, "cityblock").build_graph(16, 16)
    with pytest.raises(ValueError):
        ItemIndex(torch.randn(60, 8, device=DEV), "L2").build_graph(16, 64)


# ---------------------------------------------------------------------------------------------------- search
def _int_case(metric, n=1500, dim=12, d=16, D=32, seed=0):
    rng = np.random.default_rng(seed)
    table = X.small_ints(rng, (n, dim))
    queries = X.small_ints(rng, (12, dim))
    index = ItemIndex(torch.from_numpy(table).to(DEV), metric).build_graph(d, D)
    return table, queries, index


def _replay(index, table, queries, metric, T, W, M, k, exclude=None, buffers=None):
    keys = X.keys32(X.scores64(queries, table), X.norms32(table, metric), metric).numpy()
    qn = X.qnorm32(queries)
    finish = lambda r, kk: X.finish32(torch.from_numpy(kk)[None], qn[r:r + 1], metric)[0].numpy()
    pad = X.FLT_MAX if metric == "L2" else -X.FLT_MAX
    return G.search(keys, _np(index.graph), _np(index.graph_entry), T, W, M, k, finish, pad, exclude, buffers)


@pytest.mark.parametrize("M", [0, 3])
@pytest.mark.parametrize("W", [1, 4])
@pytest.mark.parametrize("T", [32, 64, 256])
@pytest.mark.parametrize("metric", METRICS)
def test_search_matches_replay(metric, T, W, M):
    table, queries, index = _int_case(metric)
    param = {"itopk_size": T, "search_width": W, "max_iterations": M}
    rng = np.random.default_rng(T + W)
    excl = [rng.choice(1500, 40, replace=False).tolist() if r % 3 else None for r in range(len(queries))]
    keys = X.keys32(X.scores64(queries, table), X.norms32(table, metric), metric).numpy()
    bufs = [G.replay(keys[r], _np(index.graph), _np(index.graph_entry), T, W, M) for r in range(len(queries))]
    for k in [1, 10, 64]:
        if k > T:
            continue
        for ex in [None, excl]:
            want_i, want_d, want_it = _replay(index, table, queries, metric, T, W, M, k, ex, bufs)
            sets = None if ex is None else ItemSets.from_lists([x or [] for x in ex], device=DEV)
            res = index.search(torch.from_numpy(queries).to(DEV), k, search_param=param, exclude=sets)
            np.testing.assert_array_equal(_np(res.ids), want_i, err_msg="k %d exclude %s" % (k, ex is not None))
            np.testing.assert_array_equal(_np(res.distances), want_d)
    it = index.graph_iterations(torch.from_numpy(queries).to(DEV), param)
    np.testing.assert_array_equal(_np(it), want_it)
    if M:
        assert int(it.max()) <= M


_CLEAR_CASES = {}


def _clear_case(metric):
    """20,000 small-integer items, d = D = 64: a wide search keys several thousand ids, so the visited hash (2,048
    ids) is cleared and refilled during every query"""
    if metric not in _CLEAR_CASES:
        _CLEAR_CASES.clear()
        rng = np.random.default_rng(21)
        table, queries = X.small_ints(rng, (20000, 12)), X.small_ints(rng, (8, 12))
        index = ItemIndex(torch.from_numpy(table).to(DEV), metric).build_graph(64, 64)
        _CLEAR_CASES[metric] = (table, queries, index)
    return _CLEAR_CASES[metric]


@pytest.mark.parametrize("T,W", [(256, 4), (128, 4), (256, 8)])
@pytest.mark.parametrize("metric", METRICS)
def test_search_matches_replay_across_hash_clears(metric, T, W):
    table, queries, index = _clear_case(metric)
    graph, entry = _np(index.graph), _np(index.graph_entry)
    keys = X.keys32(X.scores64(queries, table), X.norms32(table, metric), metric).numpy()
    clears = [G.hash_clears(keys[r], graph, entry, T, W) for r in range(len(queries))]
    assert min(clears) >= 1 and max(clears) >= 2, clears
    bufs = [G.replay(keys[r], graph, entry, T, W) for r in range(len(queries))]
    rng = np.random.default_rng(T + W)
    # exclude some of each query's own best items, so exclusion acts on entries the traversal kept
    excl = [[i for _, i in bufs[r][0][:T:3]] + rng.choice(20000, 50, replace=False).tolist() if r % 2 else None
            for r in range(len(queries))]
    param = {"itopk_size": T, "search_width": W}
    q = torch.from_numpy(queries).to(DEV)
    for k in [10, 64]:
        for ex in [None, excl]:
            want_i, want_d, want_it = _replay(index, table, queries, metric, T, W, 0, k, ex, bufs)
            sets = None if ex is None else ItemSets.from_lists([x or [] for x in ex], device=DEV)
            res = index.search(q, k, search_param=param, exclude=sets)
            np.testing.assert_array_equal(_np(res.ids), want_i, err_msg="k %d exclude %s" % (k, ex is not None))
            np.testing.assert_array_equal(_np(res.distances), want_d)
    np.testing.assert_array_equal(_np(index.graph_iterations(q, param)), want_it)


@pytest.mark.parametrize("metric", METRICS)
def test_full_coverage_is_the_flat_search(metric):
    rng = np.random.default_rng(11)
    table, queries = X.small_ints(rng, (200, 10)), X.small_ints(rng, (20, 10))
    index = ItemIndex(torch.from_numpy(table).to(DEV), metric).build_graph(16, 32)
    q = torch.from_numpy(queries).to(DEV)
    got = index.search(q, 64, search_param={"itopk_size": 256})
    flat = ItemIndex(torch.from_numpy(table).to(DEV), metric).search(q, 64)
    assert torch.equal(got.ids, flat.ids) and torch.equal(got.distances, flat.distances)
    want_i, want_d = X.topk(queries, table, metric, 64)
    np.testing.assert_array_equal(_np(got.ids), want_i)


@pytest.mark.parametrize("metric", METRICS)
def test_batch_invariance(metric):
    table = torch.randn(5000, 40, device=DEV, generator=torch.Generator(device=DEV).manual_seed(3))
    index = ItemIndex(table, metric).build_graph(32, 64)
    q = torch.randn(70, 40, device=DEV, generator=torch.Generator(device=DEV).manual_seed(4))
    param = {"itopk_size": 64, "search_width": 2}
    full = index.search(q, 10, search_param=param)
    for sl in [slice(0, 1), slice(5, 12), slice(33, 70)]:
        part = index.search(q[sl], 10, search_param=param)
        assert torch.equal(part.ids, full.ids[sl]) and torch.equal(part.distances, full.distances[sl])


def test_search_param_validation():
    table, queries, index = _int_case("L2", n=300)
    q = torch.from_numpy(queries).to(DEV)
    for bad in [{"nprobe": 4}, {"itopk_size": 48}, {"itopk_size": 512}, {"search_width": 0}, {"search_width": 9},
                {"max_iterations": -1}]:
        with pytest.raises(ValueError):
            index.search(q, 10, search_param=bad)
    with pytest.raises(ValueError):
        index.search(q, 64, search_param={"itopk_size": 32})
    index.search(q, 10)                                          # the defaults: T 64, W 1, M 0


# The replay's recall@10 at test-writing time on this mixture (20,000 x 64 items, 100 overlapping components with
# N(0, 1) centres and N(0, 1) spread, 200 queries from the same mixture, L2, d 32 / D 64, exact k-NN): 0.988 at T 64,
# W 1 and 0.978 at T 32, W 1.  Float keys, so the device may differ from the replay in the last bits; the floor leaves
# room for that.  (Components that do not overlap are the case a k-NN graph cannot serve: every list stays inside its
# component and a search reaches only the components of its entry points.)
RECALL_FLOOR = 0.95


def test_recall_floor_on_a_mixture():
    x = _mixture(20000 + 200, 64, 100, 0)
    table, q = torch.from_numpy(x[:20000]).to(DEV), torch.from_numpy(x[20000:]).to(DEV)
    index = ItemIndex(table, "L2").build_graph(32, 64)
    exact = ItemIndex(table, "L2").search(q, 10).ids
    got = index.search(q, 10, search_param={"itopk_size": 64, "search_width": 1}).ids
    _, mean = recall_at_k(got, exact)
    print("graph recall@10 on the mixture at T 64, W 1: %.3f" % mean)
    assert mean >= RECALL_FLOOR


def test_long_traversal_262144_items():
    rng = np.random.default_rng(12)
    n = 262144
    table, queries = X.small_ints(rng, (n, 8), -4, 4), X.small_ints(rng, (4, 8), -4, 4)
    index = ItemIndex(torch.from_numpy(table).to(DEV), "L2").build_graph(32, 32)
    param = {"itopk_size": 64, "search_width": 1}
    got = index.search(torch.from_numpy(queries).to(DEV), 10, search_param=param)
    tt = torch.from_numpy(table).to(DEV)
    keys = X.keys32(X.scores64(torch.from_numpy(queries).to(DEV), tt), X.norms32(tt, "L2"), "L2").cpu().numpy()
    qn = X.qnorm32(queries)
    finish = lambda r, kk: X.finish32(torch.from_numpy(kk)[None], qn[r:r + 1], "L2")[0].numpy()
    want_i, want_d, iters = G.search(keys, _np(index.graph), _np(index.graph_entry), 64, 1, 0, 10, finish, X.FLT_MAX)
    np.testing.assert_array_equal(_np(got.ids), want_i)
    np.testing.assert_array_equal(_np(got.distances), want_d)
    print("iterations to convergence: %s" % iters.tolist())


# ---------------------------------------------------------------------------------------------------- persistence
@pytest.mark.parametrize("metric", METRICS)
def test_state_round_trip(metric):
    table = torch.randn(2000, 24, device=DEV, generator=torch.Generator(device=DEV).manual_seed(5))
    a = ItemIndex(table, metric).build_graph(16, 32)
    state = a.graph_state()
    b = ItemIndex(table, metric).load_graph(state)
    assert torch.equal(a.graph, b.graph) and torch.equal(a.graph_entry, b.graph_entry)
    q = torch.randn(9, 24, device=DEV)
    ra, rb = a.search(q, 10), b.search(q, 10)
    assert torch.equal(ra.ids, rb.ids) and torch.equal(ra.distances, rb.distances)
    assert ItemIndex(table, metric).build_ivf(8).load_graph(state).ivf is None


def test_load_refuses_corrupted_state():
    table = torch.randn(500, 16, device=DEV)
    state = ItemIndex(table, "L2").build_graph(16, 32).graph_state()

    def corrupt(fn):
        s = {k: (v.clone() if torch.is_tensor(v) else v) for k, v in state.items()}
        fn(s)
        return s
    bad = [corrupt(lambda s: s["graph"].__setitem__((3, 0), 3)),                    # self-loop
           corrupt(lambda s: s["graph"].__setitem__((4, 1), int(s["graph"][4, 0]))),  # repeated id
           corrupt(lambda s: s["graph"].__setitem__((5, 2), 500)),                  # out of range
           corrupt(lambda s: s["entry"].__setitem__(0, -1)),
           corrupt(lambda s: s.__setitem__("graph", s["graph"][:, :12].contiguous())),
           corrupt(lambda s: s.__setitem__("graph", s["graph"].long())),
           corrupt(lambda s: s.__setitem__("metric", "IP")),
           corrupt(lambda s: s.__setitem__("n_items", 499)),
           {"graph": state["graph"]}]
    for s in bad:
        with pytest.raises(ValueError):
            ItemIndex(table, "L2").load_graph(s)


def test_milvus_connection_builds_cagra():
    x = torch.randn(500, 16, device=DEV)
    conn = MilvusConnection(x, param={"index_type": "GPU_CAGRA", "intermediate_graph_degree": 32, "graph_degree": 16})
    assert conn.graph is not None and conn.graph.shape == (500, 16)
    assert MilvusConnection(x, param={"index_type": "GPU_CAGRA"}).graph.shape == (500, 32)
    with pytest.raises(ValueError, match="k is at most 64"):
        MilvusConnection(x, param={"index_type": "GPU_CAGRA", "intermediate_graph_degree": 128})


# ---------------------------------------------------------------------------------------------------- workspace contract
@pytest.mark.parametrize("d,D", [(16, 32), (64, 64)])
def test_workspace_bounds_build(d, D):
    n = 3001
    table = torch.randn(n, 20, device=DEV)
    knn = ItemIndex(table, "L2").knn_lists(D)
    entry = torch.arange(512, dtype=torch.int32, device=DEV)

    def run(w, nbytes):
        index = _lib.graph_index(n, 20, _lib.METRIC_L2, d, None, None, w["graph"], entry)
        args = _lib.GraphBuildArgs(index, knn.data_ptr(), D, 0, _ptr(w, "flag"), _ptr(w, "ws"), nbytes)
        return L.recnn_graph_build(ctypes.byref(args), _lib.stream_ptr())
    sizes = dict(ws=L.recnn_graph_build_workspace_bytes(n, d), graph=n * d * 4, flag=4)
    check_windows(sizes, [(True, run)])


@pytest.mark.parametrize("T,W", [(32, 1), (256, 4)])
@pytest.mark.parametrize("dim,metric", [(13, "COS"), (64, "L2"), (132, "IP")])
def test_workspace_bounds_search(dim, metric, T, W):
    table = torch.randn(4000, dim, device=DEV, generator=torch.Generator(device=DEV).manual_seed(dim))
    index = ItemIndex(table, metric).build_graph(16, 32)
    nq, k = 40, 17
    qs = torch.randn(nq, dim, device=DEV)
    sets, flag = set_table(nq, 4000, dim), torch.zeros(1, dtype=torch.int32, device=DEV)

    def run(with_sets):
        def go(w, nbytes):
            sa = set_args(sets) if with_sets else (None, 0, None, 0, None)
            args = _lib.GraphSearchArgs(index._graph_descriptor(index._graph), qs.data_ptr(), nq, k, T, W, 0, *sa,
                                        _ptr(w, "ids"), _ptr(w, "dist"), _ptr(w, "iters"),
                                        flag.data_ptr() if with_sets else None, _ptr(w, "ws"), nbytes)
            return L.recnn_graph_search(ctypes.byref(args), _lib.stream_ptr())
        return go
    sizes = dict(ws=L.recnn_graph_search_workspace_bytes(nq, T), ids=nq * k * 8, dist=nq * k * 4, iters=nq * 4)
    check_windows(sizes, [(True, run(False))])
    check_windows(sizes, [(True, run(True))], [flag], [flag])
