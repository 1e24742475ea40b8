"""ItemIndex under the scipy.spatial.distance metrics on the device (the CUDA-core distance kernel of distance.cuh
behind recnn_retrieve_topk / _rank and their *_sets forms).

Cityblock, Chebyshev, Canberra and Bray-Curtis fix their accumulation order, so ids and distances equal the fp32 replay
(tests/_metric_oracle.py) bit for bit, on small integers and on Gaussians alike.  Correlation rounds differently from
the replay's fma-through-float64, so it is held to float64 within a bar derived from its fp32 error."""
from __future__ import annotations

import numpy as np
import pytest
import torch

from recnn_b200 import _lib
from recnn_b200.data import ItemSets
from recnn_b200.data.db_con import ItemIndex
from tests import _metric_oracle as M
from tests.test_workspace_bounds_serving_gpu import KS, _flag, _ptr, check_windows, set_args, set_table

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda")
CODE = {name: getattr(_lib, "METRIC_" + code) for code, name in M.NAME.items()}

# (dim, n_items, k, n_queries, kind): every dim of 1, 3, 13, 64, 130, 257 (1 and 3 are shorter than one 8-wide d
# chunk; 130 and 257 end in a partial one), every n_items of 1, 127, 5,003, 70,000 (above 65,536 items a slab is 128
# queries, so 260 and 200 queries take three and two slabs), every k of 1, 10, 64
CASES = [(1, 1, 1, 5, "ints"), (3, 127, 10, 33, "ints"), (13, 127, 64, 7, "gauss"), (64, 5003, 10, 50, "gauss"),
         (130, 5003, 64, 20, "ints"), (257, 5003, 1, 9, "gauss"), (64, 70000, 10, 260, "gauss"),
         (13, 70000, 64, 200, "ints"), (257, 70000, 1, 130, "ints")]


def _data(rng, shape, kind):
    x = M.small_ints(rng, shape) if kind == "ints" else rng.standard_normal(shape).astype(np.float32)
    return torch.from_numpy(x).to(DEV)


def _unaligned(x):
    """a contiguous copy of x that starts 4 bytes past a 16-byte boundary"""
    buf = torch.empty(x.numel() + 4, dtype=torch.float32, device=DEV)
    v = buf[1:1 + x.numel()].view(x.shape)
    v.copy_(x)
    assert v.data_ptr() % 16 == 4
    return v


def _case(seed, dim, n_items, nq, kind, unaligned=False):
    rng = np.random.default_rng(seed)
    table, q = _data(rng, (n_items, dim), kind), _data(rng, (nq, dim), kind)
    return (_unaligned(table), _unaligned(q)) if unaligned else (table, q)


@pytest.mark.parametrize("case", range(len(CASES)))
@pytest.mark.parametrize("code", M.EXACT)
def test_exact_metrics_equal_the_replay_bit_for_bit(code, case):
    dim, n_items, k, nq, kind = CASES[case]
    table, q = _case(case * 7 + len(code), dim, n_items, nq, kind, unaligned=case % 2 == 1)
    idx = ItemIndex(table, M.NAME[code])
    assert idx.table.data_ptr() % 16 == (4 if case % 2 else 0)
    res = idx.search(q, k)
    ids, dist = M.topk(q, table, code, k)
    np.testing.assert_array_equal(res.ids.cpu().numpy(), ids)
    np.testing.assert_array_equal(res.distances.cpu().numpy(), dist)


def _corr_check(q, table, ids, dist):
    """ids / dist of a search against float64: each distance within the bar of its pair, and every id where the order is
    unambiguous under the bar"""
    d64 = M.dist64(q, table, "CORR")
    bar = M.corr_bar(q, table)
    ids, dist = ids.long(), dist.double()
    np.testing.assert_array_less((dist - torch.gather(d64, 1, ids)).abs().cpu(), torch.gather(bar, 1, ids).cpu() + 1e-300)
    k = ids.shape[1]
    order = torch.sort(d64, dim=1, stable=True).indices[:, :k]
    # the returned set is the true top k up to the bar
    kth = torch.gather(d64, 1, order[:, -1:])
    assert bool((torch.gather(d64, 1, ids) <= kth + 2 * bar.amax(1, keepdim=True)).all())
    for r in range(ids.shape[0]):
        for i in range(k):
            j = int(order[r, i])
            others = torch.cat([d64[r, :j], d64[r, j + 1:]])
            if others.numel() == 0 or (others - d64[r, j]).abs().min() > 2 * bar[r].max():
                assert int(ids[r, i]) == j, (r, i)


@pytest.mark.parametrize("dim,n_items,k,nq,offset", [(3, 127, 10, 33, 0.0), (64, 5003, 64, 20, 100.0),
                                                    (257, 70000, 10, 130, 3.0), (13, 70000, 1, 200, 0.0)])
def test_correlation_against_float64(dim, n_items, k, nq, offset):
    table, q = _case(dim, dim, n_items, nq, "gauss", unaligned=dim % 2 == 1)
    table, q = table + offset, q - offset                 # a large mean: the centring must not cancel
    idx = ItemIndex(table, "correlation")
    res = idx.search(q, k)
    _corr_check(q, table, res.ids, res.distances)


def test_correlation_constant_rows_are_at_distance_one():
    rng = np.random.default_rng(5)
    table = torch.from_numpy(rng.standard_normal((300, 9)).astype(np.float32)).to(DEV)
    table[[3, 40, 41]] = torch.tensor([0.1, 0.0, -7.0], device=DEV)[:, None]     # 0.1: its fp32 sum/9 is not 0.1
    q = torch.from_numpy(rng.standard_normal((4, 9)).astype(np.float32)).to(DEV)
    q[1] = 0.1
    q[2] = 0.0
    idx = ItemIndex(table, "correlation")
    res = idx.search(q, 64)
    # a constant query is at 1 from every item: the first 64 ids, all at 1
    for r in (1, 2):
        assert res.ids[r].tolist() == list(range(64))
        assert bool((res.distances[r] == 1).all())
    # constant items are at exactly 1 from every query: their rank equals the count of items strictly closer than 1
    d = M.dist64(q, table, "CORR")
    for r in (0, 3):
        for j in (3, 40, 41):
            rk = int(idx.rank(q[r:r + 1], torch.tensor([j], device=DEV))[0])
            assert rk == int((d[r] < 1).sum()) + int(((d[r] == 1) & (torch.arange(300, device=DEV) < j)).sum())


@pytest.mark.parametrize("name", list(M.NAME.values()))
def test_rank_is_the_replay_count_and_the_search_position(name):
    code = {v: k for k, v in M.NAME.items()}[name]
    nq, n_items, dim = 150, 70000, 13                      # two slabs
    table, q = _case(21, dim, n_items, nq, "ints")
    idx = ItemIndex(table, name)
    rng = np.random.default_rng(22)
    res = idx.search(q, 64)
    # targets: half from the top 64 (their position must be the rank), half anywhere
    pick = torch.from_numpy(rng.integers(0, 64, nq)).to(DEV)
    target = torch.gather(res.ids, 1, pick[:, None])[:, 0]
    target[::2] = torch.from_numpy(rng.integers(0, n_items, nq)[::2]).to(DEV)
    lists = [np.sort(rng.choice(n_items, 40, replace=False)) for _ in range(nq)]
    lists = [l[l != int(t)] for l, t in zip(lists, target.tolist())]
    sets = ItemSets.from_lists(lists, device=DEV)
    for exclude in (None, sets):
        rk = idx.rank(q, target, exclude=exclude)
        top = idx.search(q, 64, exclude=exclude).ids
        if code != "CORR":
            np.testing.assert_array_equal(rk.cpu().numpy(), M.rank(q, table, code, target.cpu().numpy(),
                                                                   None if exclude is None else lists))
        for r in range(nq):
            hit = (top[r] == target[r]).nonzero()
            if int(rk[r]) < 64:
                assert hit.numel() == 1 and int(hit[0]) == int(rk[r])
            else:
                assert hit.numel() == 0


@pytest.mark.parametrize("code", M.EXACT)
def test_exclusion_equals_the_replay_without_the_excluded(code):
    nq, n_items, dim, k = 140, 70000, 13, 64
    table, q = _case(31, dim, n_items, nq, "gauss", unaligned=True)
    idx = ItemIndex(table, M.NAME[code])
    rng = np.random.default_rng(32)
    # shared sets through exclude_rows (one longer than the 4,096 ids staged in shared memory; -1: none)
    shared = [np.sort(rng.choice(n_items, m, replace=False)) for m in (5000, 30, 1)]
    rows = np.array([-1 if r % 4 == 3 else r % 3 for r in range(nq)], np.int64)
    got = idx.search(q, k, exclude=ItemSets.from_lists(shared, device=DEV), exclude_rows=torch.from_numpy(rows))
    want = M.topk(q, table, code, k, exclude=[shared[s] if s >= 0 else [] for s in rows])
    np.testing.assert_array_equal(got.ids.cpu().numpy(), want[0])
    np.testing.assert_array_equal(got.distances.cpu().numpy(), want[1])
    # one list per query, some holding the query's best items
    base = M.topk(q, table, code, 8)[0]
    lists = [np.concatenate([base[r, :r % 9], rng.choice(n_items, 20)]) for r in range(nq)]
    got = idx.search(q, k, exclude=ItemSets.from_lists(lists, device=DEV))
    want = M.topk(q, table, code, k, exclude=lists)
    np.testing.assert_array_equal(got.ids.cpu().numpy(), want[0])
    np.testing.assert_array_equal(got.distances.cpu().numpy(), want[1])


def test_exclusion_pads_short_rows_with_flt_max():
    table, q = _case(33, 5, 20, 3, "gauss")
    for name in list(M.NAME.values()) + ["euclidean", "cosine"]:
        res = ItemIndex(table, name).search(q, 10, exclude=ItemSets.from_lists([range(12), [], range(20)], device=DEV))
        assert res.ids[0, 8:].tolist() == [-1, -1] and bool((res.ids[1] >= 0).all())
        assert res.ids[2].tolist() == [-1] * 10
        assert bool((res.distances[0, 8:] == M.FLT_MAX).all()) and bool((res.distances[2] == M.FLT_MAX).all())


@pytest.mark.parametrize("name", list(M.NAME.values()))
def test_a_query_does_not_depend_on_its_batch(name):
    nq, n_items, dim = 300, 70000, 24                     # three slabs of 128
    table, q = _case(41, dim, n_items, nq, "gauss")
    idx = ItemIndex(table, name)
    full = idx.search(q, 10)
    for r in (0, 127, 128, 299):
        alone = idx.search(q[r:r + 1], 10)
        assert torch.equal(alone.ids[0], full.ids[r]) and torch.equal(alone.distances[0], full.distances[r])
    part = idx.search(q[100:230], 10)
    assert torch.equal(part.ids, full.ids[100:230]) and torch.equal(part.distances, full.distances[100:230])
    rk = idx.rank(q, full.ids[:, 3])
    assert torch.equal(rk[5:6], idx.rank(q[5:6], full.ids[5:6, 3]))


@pytest.mark.parametrize("name", list(M.NAME.values()))
def test_non_finite_rows_rank_after_finite_and_before_padding(name):
    code = {v: k for k, v in M.NAME.items()}[name]
    rng = np.random.default_rng(51)
    n_items, dim = 40, 6
    table = torch.from_numpy(rng.standard_normal((n_items, dim)).astype(np.float32)).to(DEV)
    table[7, 2] = float("nan")
    table[11] = 3e38                                      # |q - t| sums, |q + t| and the mean overflow
    table[12] = -3e38
    q = torch.from_numpy(rng.standard_normal((3, dim)).astype(np.float32)).to(DEV)
    q[2, 0] = 3e38
    bad = {7, 11, 12}
    ex = ItemSets.from_lists([[j for j in range(n_items) if j not in bad and j % 3]] * 3, device=DEV)
    res = ItemIndex(table, name).search(q, 20, exclude=ex)
    ids, dist = res.ids.cpu().numpy(), res.distances.cpu().numpy()
    for r in range(3):
        live = ids[r][ids[r] >= 0]
        assert (ids[r][len(live):] == -1).all() and len(live) == n_items - len(ex.set(r))
        flt = dist[r][:len(live)] == M.FLT_MAX
        # every FLT_MAX entry comes after every finite one, in id order, and NaN rows are among them
        assert flt[flt.argmax():].all() if flt.any() else True
        assert list(live[flt]) == sorted(live[flt]) and 7 in set(live[flt])
        assert np.isfinite(dist[r][:len(live)]).all()
    if code != "CORR":
        want = M.topk(q, table, code, 20, exclude=[ex.set(r).cpu().numpy() for r in range(3)])
        np.testing.assert_array_equal(ids, want[0])
        np.testing.assert_array_equal(dist, want[1])


def test_scipy_names_on_l2_and_cos():
    table, q = _case(61, 32, 5003, 40, "gauss")
    l2, cos = ItemIndex(table, "L2").search(q, 10), ItemIndex(table, "COS").search(q, 10)
    for name, p in (("euclidean", None), ("minkowski", None), ("minkowski", 2)):
        res = ItemIndex(table, name, p=p).search(q, 10)
        assert torch.equal(res.ids, l2.ids) and torch.equal(res.distances, torch.sqrt(l2.distances))
    res = ItemIndex(table, "cosine").search(q, 10)
    assert torch.equal(res.ids, cos.ids) and torch.equal(res.distances, torch.clamp(1 - cos.distances, 0, 2))
    np.testing.assert_allclose(res.distances.cpu().numpy(),
                               np.take_along_axis(M.scipy_dist(q, table, "cosine"), res.ids.cpu().numpy(), 1),
                               rtol=0, atol=1e-5)
    for p, name in ((1, "cityblock"), (float("inf"), "chebyshev")):
        a, b = ItemIndex(table, "minkowski", p=p).search(q, 10), ItemIndex(table, name).search(q, 10)
        assert torch.equal(a.ids, b.ids) and torch.equal(a.distances, b.distances)
    # ranks are the L2 / COS ranks
    target = l2.ids[:, 4]
    assert torch.equal(ItemIndex(table, "euclidean").rank(q, target), ItemIndex(table, "L2").rank(q, target))


@pytest.mark.parametrize("name", M.SCIPY_NAMES)
def test_demo_ranking_on_small_ints(name):
    """ItemIndex(table, name).search(action, k) against the demo's sorted(items, key=metric)[:k] on {-1, 0, 1}
    entries (exact in fp32 for all but cosine and correlation, which must agree where scipy's order is unambiguous)"""
    from scipy.spatial import distance
    rng = np.random.default_rng(71)
    table, q = M.small_ints(rng, (400, 16), -1, 1), M.small_ints(rng, (3, 16), -1, 1)
    res = ItemIndex(torch.from_numpy(table).to(DEV), name).search(torch.from_numpy(q).to(DEV), 10)
    f = getattr(distance, name)
    exact = M.scipy_dist(q, table, name)
    for r in range(len(q)):
        demo = sorted(range(len(table)), key=lambda j: f(table[j].astype(np.float64), q[r].astype(np.float64)))[:10]
        got = res.ids[r].cpu().numpy()
        np.testing.assert_allclose(res.distances[r].cpu().numpy(), exact[r, got], rtol=1e-6, atol=1e-5)
        if name not in ("cosine", "correlation"):
            assert list(got) == demo
        else:
            np.testing.assert_allclose(exact[r, got], exact[r, demo], rtol=0, atol=1e-5)


# ---------------------------------------------------------------- the workspace contract
# (queries, items, dim): 130 queries over 70,001 items take two slabs of 128 that reuse the distances and partials
METRIC_WS = [(130, 70001, 13), (9, 1000, 130)]


def _norms(table, metric):
    if metric != _lib.METRIC_CORR:
        return None
    items, dim = table.shape
    norms = torch.empty(2 * items, device=DEV)
    _lib.check(_lib.lib().recnn_item_norms(table.data_ptr(), items, dim, metric, norms.data_ptr(), _lib.stream_ptr()))
    return norms


@pytest.mark.parametrize("metric", sorted(CODE.values()))
@pytest.mark.parametrize("nq,items,dim", METRIC_WS)
def test_workspace_exact_size(nq, items, dim, metric):
    L = _lib.lib()
    torch.manual_seed(items + dim + metric)
    table = _unaligned(torch.randn(items, dim, device=DEV))
    queries = _unaligned(torch.randn(nq, dim, device=DEV))
    norms = _norms(table, metric)
    sets, flag = set_table(nq, items, dim), _flag()
    target = torch.randint(0, items, (nq,), device=DEV)
    for k in KS:
        def topk(w, nbytes):
            return L.recnn_retrieve_topk_sets(queries.data_ptr(), nq, dim, table.data_ptr(), items, _lib.ptr(norms),
                                              metric, k, *set_args(sets), _ptr(w, "ids"), _ptr(w, "dist"),
                                              flag.data_ptr(), _ptr(w, "ws"), nbytes, _lib.stream_ptr())
        sizes = dict(ws=L.recnn_retrieve_workspace_bytes(nq, items, k), ids=nq * k * 8, dist=nq * k * 4)
        check_windows(sizes, [(True, topk)], [flag], [flag])
    head = (queries.data_ptr(), nq, dim, table.data_ptr(), items, _lib.ptr(norms), metric, target.data_ptr())

    def rank(w, nbytes):
        return L.recnn_retrieve_rank_sets(*head, *set_args(sets), _ptr(w, "rank"), flag.data_ptr(), _ptr(w, "ws"),
                                          nbytes, _lib.stream_ptr())
    check_windows(dict(ws=L.recnn_retrieve_rank_workspace_bytes(nq, items), rank=nq * 8), [(True, rank)], [flag],
                  [flag])


def test_item_norms_of_correlation():
    rng = np.random.default_rng(81)
    table = torch.from_numpy(rng.standard_normal((1000, 37)).astype(np.float32) + 5).to(DEV)
    table[3] = 0.1
    norms = _norms(_unaligned(table), _lib.METRIC_CORR)
    mean, cn = M.corr_stats32(table)
    assert torch.equal(norms[:1000], mean)                 # the ascending fp32 sum / dim, bit for bit
    torch.testing.assert_close(norms[1000:], cn, rtol=1e-6, atol=0)
    assert norms[3] == table[3, 0] and norms[1003] == 0
