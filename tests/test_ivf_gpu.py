"""IVF_FLAT on the device (recnn_ivf_build / recnn_ivf_search behind ItemIndex.build_ivf and search) against the float64
oracle of tests/_ivf_oracle.py.  dim 64 and 132 run the coarse and assignment searches on the tensor-core GEMM, dim 13 on
the CUDA-core one; the fine scan is the same kernel at every dim."""
from __future__ import annotations

import ctypes

import numpy as np
import pytest
import torch

from recnn_b200 import _lib
from recnn_b200.data import ItemIndex, ItemSets, MilvusConnection
from recnn_b200.utils.metrics import recall_at_k
from tests import _ivf_oracle as V
from tests.test_workspace_bounds_serving_gpu import check_windows, _ptr, set_args, set_table

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
L = _lib.lib()
METRICS = ["L2", "IP", "COS"]
DIMS = [13, 64, 132]


def _dev(x):
    return torch.from_numpy(np.ascontiguousarray(x, dtype=np.float32)).to(DEV)


def _np(t):
    return t.detach().cpu().numpy()


def _blobs(dim, n_blobs, n_per, seed):
    rng = np.random.default_rng(seed)
    centers = rng.standard_normal((n_blobs, dim))
    centers = 10.0 * centers / np.linalg.norm(centers, axis=1, keepdims=True)
    x, labels = V.blobs(n_per, centers, 0.2, seed + 1)
    return x.astype(np.float32), labels


def _blobs_covering(dim, n_blobs, n_per, seed):
    """blobs with the rows ordered so that seed 0's initial centroids are one point of each blob: Lloyd then converges to
    the blobs, and no assignment is a near-tie"""
    x, labels = _blobs(dim, n_blobs, n_per, seed)
    _, init = V.sample_plan(len(x), n_blobs, 0)
    firsts = np.arange(n_blobs) * n_per
    order = np.empty(len(x), np.int64)
    order[init] = firsts
    order[np.setdiff1d(np.arange(len(x)), init)] = np.setdiff1d(np.arange(len(x)), firsts)
    return x[order], labels[order]


def _values64(queries, table, ids, metric):
    """float64 distance / similarity of each (query, id) as recnn_retrieve_topk reports it (NaN for -1)"""
    q, t = np.asarray(queries, np.float64), np.asarray(table, np.float64)
    out = np.full(ids.shape, np.nan)
    for r in range(len(q)):
        ok = ids[r] >= 0
        x = t[ids[r][ok]]
        if metric == "L2":
            v = ((x - q[r]) ** 2).sum(1)
        elif metric == "IP":
            v = x @ q[r]
        else:
            v = (x @ q[r]) / np.maximum(np.linalg.norm(x, axis=1), 1e-30) / max(np.linalg.norm(q[r]), 1e-30)
        out[r, ok] = v
    return out


def _tol(queries, table, metric):
    qn = np.linalg.norm(np.asarray(queries, np.float64), axis=1).max()
    tn = np.linalg.norm(np.asarray(table, np.float64), axis=1).max()
    scale = {"L2": (qn + tn) ** 2, "IP": qn * tn, "COS": 1.0}[metric]
    return 2e-5 * scale


def check_topk(got_i, got_d, want_i, want_d, queries, table, metric):
    """device ids / distances against the float64 top-k of the same candidate sets: the reported distances are the
    float64 values of the returned ids within fp32 tolerance, they match the oracle's sequence, and the ids are the
    oracle's wherever the oracle's value is clear of its neighbours (a near-tie may swap)"""
    tol = _tol(queries, table, metric)
    assert (got_i == -1).sum() == (want_i == -1).sum()
    pad = want_i == -1
    np.testing.assert_array_equal(got_i[pad], -1)
    v = _values64(queries, table, got_i, metric)
    np.testing.assert_allclose(got_d[~pad], v[~pad], atol=tol, rtol=0)
    np.testing.assert_allclose(got_d[~pad], want_d[~pad], atol=2 * tol, rtol=0)
    for r in range(len(want_i)):
        nf = int((want_i[r] >= 0).sum())
        w = want_d[r, :nf]
        for j in range(nf - 1):                                   # the last may tie with the first item past k
            if (np.abs(np.delete(w, j) - w[j]) > 2 * tol).all():
                assert got_i[r, j] == want_i[r, j], (r, j, got_i[r], want_i[r])


def _device_probes(index, queries, nprobe):
    """the lists the device probed: the coarse step is recnn_retrieve_topk over the centroids, as a flat ItemIndex"""
    coarse = ItemIndex(index.ivf.centroids, index.metric_name)
    return _np(coarse.search(queries, nprobe).ids)


def _lists(index):
    iv = index.ivf
    return _np(iv.centroids).astype(np.float64), _np(iv.list_offsets), _np(iv.list_ids)


# ---------------------------------------------------------------------------------------------------- build
@pytest.mark.parametrize("dim", DIMS)
@pytest.mark.parametrize("metric", METRICS)
def test_build_matches_oracle_on_blobs(metric, dim):
    nlist = 16
    x, labels = _blobs_covering(dim, nlist, 150, 10 + dim)
    index = ItemIndex(_dev(x), metric).build_ivf(nlist, n_iter=8, seed=0)
    c, offsets, ids = _lists(index)
    wc, woffsets, wids = V.build(x, metric, nlist, n_iter=8, seed=0)
    np.testing.assert_array_equal(offsets, woffsets)
    np.testing.assert_array_equal(ids, wids)
    np.testing.assert_allclose(c, wc, atol=1e-5 * np.abs(wc).max(), rtol=0)
    assert sorted(tuple(ids[offsets[l]:offsets[l + 1]]) for l in range(nlist)) == \
        sorted(tuple(np.nonzero(labels == b)[0]) for b in range(nlist))


@pytest.mark.parametrize("dim", DIMS)
@pytest.mark.parametrize("metric", METRICS)
def test_build_invariants_on_iid_data(metric, dim):
    rng = np.random.default_rng(dim)
    x = rng.standard_normal((6000, dim)).astype(np.float32)
    index = ItemIndex(_dev(x), metric).build_ivf(48, n_iter=6, seed=1, max_points_per_centroid=64)
    c, offsets, ids = _lists(index)
    assert offsets[0] == 0 and offsets[-1] == len(x) and (np.diff(offsets) >= 0).all()
    np.testing.assert_array_equal(np.sort(ids), np.arange(len(x)))
    for l in range(48):
        seg = ids[offsets[l]:offsets[l + 1]]
        assert (np.diff(seg) > 0).all()
    item_list = np.repeat(np.arange(48), np.diff(offsets))[np.argsort(ids)]
    t = x.astype(np.float64)
    if metric == "COS":
        score = -(V._unit(t) @ V._unit(c).T)
        margin = 1e-5
    else:
        score = V.l2_keys(t, c)
        margin = 1e-5 * np.abs(score).max()
    best = score.min(1)
    gap = score[np.arange(len(x)), item_list] - best
    off = gap > 0
    assert (gap[off] <= margin).all(), "an item is not in its nearest centroid's list by %g" % gap.max()
    print("items in a near-tie list (within %g): %d of %d" % (margin, int(off.sum()), len(x)))


def test_build_is_bit_reproducible():
    rng = np.random.default_rng(5)
    x = _dev(rng.standard_normal((20000, 64)))
    a = ItemIndex(x, "L2").build_ivf(64, n_iter=5, seed=3)
    b = ItemIndex(x, "L2").build_ivf(64, n_iter=5, seed=3)
    for k in ("centroids", "centroid_norms", "list_offsets", "list_ids", "list_table", "list_norms"):
        assert torch.equal(a._ivf[k], b._ivf[k]), k
    c = ItemIndex(x, "L2").build_ivf(64, n_iter=5, seed=4)
    assert not torch.equal(a._ivf["centroids"], c._ivf["centroids"])


def test_build_refuses_bad_arguments():
    index = ItemIndex(torch.randn(100, 8, device=DEV), "L2")
    for kw in (dict(nlist=0), dict(nlist=101), dict(nlist=4, n_iter=-1), dict(nlist=4, max_points_per_centroid=0)):
        with pytest.raises(ValueError):
            index.build_ivf(**kw)
    with pytest.raises(ValueError):
        ItemIndex(torch.randn(100, 513, device=DEV), "L2").build_ivf(4)
    assert index.ivf is None


# ---------------------------------------------------------------------------------------------------- search
def _iid_index(metric, dim, n=3000, nlist=32, seed=0):
    rng = np.random.default_rng(seed + dim)
    x = rng.standard_normal((n, dim)).astype(np.float32)
    q = rng.standard_normal((40, dim)).astype(np.float32)
    return x, q, ItemIndex(_dev(x), metric).build_ivf(nlist, n_iter=5, seed=seed)


@pytest.mark.parametrize("k", [1, 10, 64])
@pytest.mark.parametrize("nprobe", [1, 4, 16])
@pytest.mark.parametrize("dim", DIMS)
@pytest.mark.parametrize("metric", METRICS)
def test_search_matches_probed_union_oracle(metric, dim, nprobe, k):
    x, q, index = _iid_index(metric, dim)
    res = index.search(_dev(q), k, search_param={"nprobe": nprobe})
    c, offsets, ids = _lists(index)
    probes = _device_probes(index, _dev(q), nprobe)
    # the device's probe choice against the float64 top-nprobe, up to near-ties of the centroid keys
    want_p = V.coarse(q, c, metric, nprobe)
    vp = _values64(q, c, probes, metric)
    wp = _values64(q, c, want_p, metric)
    np.testing.assert_allclose(np.sort(vp, 1), np.sort(wp, 1), atol=_tol(q, c, metric), rtol=0)
    want_i, want_d = V.probed_topk(q, x, metric, probes, offsets, ids, k)
    check_topk(_np(res.ids), _np(res.distances), want_i, want_d, q, x, metric)


@pytest.mark.parametrize("dim", DIMS)
@pytest.mark.parametrize("metric", METRICS)
def test_full_probe_equals_flat_search(metric, dim):
    x, q, index = _iid_index(metric, dim)
    got = index.search(_dev(q), 10, search_param={"nprobe": 32})
    flat = ItemIndex(_dev(x), metric).search(_dev(q), 10)
    want_i = _np(flat.ids)
    check_topk(_np(got.ids), _np(got.distances), want_i, _values64(q, x, want_i, metric), q, x, metric)


@pytest.mark.parametrize("metric", METRICS)
def test_batch_invariance(metric):
    x, q, index = _iid_index(metric, 64)
    qs = _dev(q)
    full = index.search(qs, 17, search_param={"nprobe": 8})
    perm = torch.randperm(len(q), generator=torch.Generator().manual_seed(0)).to(DEV)
    shuffled = index.search(qs[perm], 17, search_param={"nprobe": 8})
    assert torch.equal(shuffled.ids, full.ids[perm]) and torch.equal(shuffled.distances, full.distances[perm])
    big = torch.cat([qs, _dev(np.random.default_rng(1).standard_normal((3000, 64)))])
    many = index.search(big, 17, search_param={"nprobe": 8})
    assert torch.equal(many.ids[:len(q)], full.ids) and torch.equal(many.distances[:len(q)], full.distances)
    for r in (0, 7, len(q) - 1):
        one = index.search(qs[r:r + 1], 17, search_param={"nprobe": 8})
        assert torch.equal(one.ids[0], full.ids[r]) and torch.equal(one.distances[0], full.distances[r])


def test_search_param_and_defaults():
    x, q, index = _iid_index("L2", 16, nlist=20)
    default = index.search(_dev(q), 5)
    assert torch.equal(default.ids, index.search(_dev(q), 5, search_param={"nprobe": 16}).ids)
    for bad in ({"nprobe": 0}, {"nprobe": 21}, {"nprobe": 4, "ef": 3}, {"metric_type": "L2"}):
        with pytest.raises(ValueError):
            index.search(_dev(q), 5, search_param=bad)
    small = ItemIndex(_dev(x), "L2").build_ivf(4, n_iter=2)
    assert torch.equal(small.search(_dev(q), 5).ids, small.search(_dev(q), 5, search_param={"nprobe": 4}).ids)
    # rank stays exact
    flat = ItemIndex(_dev(x), "L2")
    target = torch.arange(len(q), device=DEV)
    assert torch.equal(index.rank(_dev(q), target), flat.rank(_dev(q), target))
    assert index.search(_dev(q[:0]), 5).ids.shape == (0, 5)


@pytest.mark.parametrize("metric", METRICS)
def test_exclusion(metric):
    x, q, index = _iid_index(metric, 64, n=2000, nlist=64)
    c, offsets, ids = _lists(index)
    probes = _device_probes(index, _dev(q), 2)
    rng = np.random.default_rng(2)
    sets = []
    for r in range(len(q)):
        union = np.concatenate([ids[offsets[l]:offsets[l + 1]] for l in probes[r]])
        if r % 4 == 0:
            sets.append(union[:max(len(union) - 3, 0)])          # fewer than k eligible: pads
        elif r % 4 == 1:
            sets.append(np.array([], np.int64))
        else:
            sets.append(rng.choice(union, min(10, len(union)), replace=False))
    ex = ItemSets.from_lists(sets, device=DEV)
    res = index.search(_dev(q), 10, search_param={"nprobe": 2}, exclude=ex)
    got_i, got_d = _np(res.ids), _np(res.distances)
    for r in range(len(q)):
        assert not set(got_i[r][got_i[r] >= 0]) & set(sets[r].tolist())
    want_i, want_d = V.probed_topk(q, x, metric, probes, offsets, ids, 10, exclude=sets)
    check_topk(got_i, got_d, want_i, want_d, q, x, metric)
    pad = got_i == -1
    assert pad[0].any()
    assert (got_d[pad] == (np.finfo(np.float32).max if metric == "L2" else -np.finfo(np.float32).max)).all()
    with pytest.raises(IndexError):
        index.search(_dev(q[:2]), 5, exclude=ItemSets.from_lists([[0, len(x)], [1]], device=DEV))
    bad = ItemSets.from_lists([[3, 1]], device=DEV)
    bad.ids = torch.tensor([3, 1], device=DEV)                     # descending: malformed
    with pytest.raises(ValueError):
        index.search(_dev(q[:1]), 5, exclude=bad)


# ---------------------------------------------------------------------------------------------------- persistence
@pytest.mark.parametrize("metric", METRICS)
def test_state_round_trip(metric):
    x, q, index = _iid_index(metric, 132)
    state = index.ivf_state()
    fresh = ItemIndex(_dev(x), metric).load_ivf(state)
    for k in ("centroids", "centroid_norms", "list_offsets", "list_ids", "list_table", "list_norms"):
        a, b = index._ivf[k], fresh._ivf[k]
        assert (a is None and b is None) or torch.equal(a, b), k
    want = index.search(_dev(q), 10, search_param={"nprobe": 4})
    got = fresh.search(_dev(q), 10, search_param={"nprobe": 4})
    assert torch.equal(want.ids, got.ids) and torch.equal(want.distances, got.distances)
    assert fresh.ivf_state()["params"] == state["params"]


def test_load_refuses_corrupted_state():
    x, q, index = _iid_index("L2", 16)
    good = index.ivf_state()

    def with_(**kw):
        s = dict(good)
        s.update(kw)
        return s
    ids, offs = good["list_ids"], good["list_offsets"]
    swapped = ids.clone()
    swapped[0] = ids[1]                                         # a repeated id: not a permutation
    descending = ids.clone()
    a, b = int(offs[0]), int(offs[1])
    descending[a:b] = ids[a:b].flip(0)
    bad_offs = offs.clone()
    bad_offs[3] = bad_offs[4] + 1                               # decreasing
    for s in (with_(list_ids=swapped), with_(list_ids=descending), with_(list_offsets=bad_offs),
              with_(list_ids=ids[:-1]), with_(metric="IP"), with_(dim=15), {"centroids": good["centroids"]}):
        with pytest.raises(ValueError):
            ItemIndex(_dev(x), "L2").load_ivf(s)


def test_milvus_connection_builds_ivf():
    x = torch.randn(500, 16, device=DEV)
    conn = MilvusConnection(x, param={"index_type": "IVF_FLAT", "nlist": 10})
    assert conn.ivf is not None and conn.ivf.centroids.shape == (10, 16)
    assert MilvusConnection(x).ivf is None
    with pytest.raises(ValueError):
        MilvusConnection(x, param={"index_type": "HNSW"})


# ---------------------------------------------------------------------------------------------------- workspace contract
@pytest.mark.parametrize("dim,metric", [(13, _lib.METRIC_COS), (64, _lib.METRIC_L2), (132, _lib.METRIC_IP)])
def test_workspace_bounds_build(dim, metric):
    n, nlist = 3001, 24
    torch.manual_seed(dim)
    table = torch.randn(n, dim, device=DEV)
    sample = torch.randperm(n, device=DEV)[:1500].contiguous()
    init = torch.randperm(1500, device=DEV)[:nlist].contiguous()
    pitch = (dim + 3) // 4 * 4
    norms = metric != _lib.METRIC_IP

    def run(w, nbytes):
        index = _lib.ivf_index(n, dim, metric, nlist, w["centroids"], w["cnorm"] if norms else None, w["offsets"],
                               w["ids"], w["table"], w["norms"] if norms else None)
        args = _lib.IvfBuildArgs(index, table.data_ptr(), sample.data_ptr(), 1500, init.data_ptr(), 4, 0,
                                 _ptr(w, "ws"), nbytes)
        return L.recnn_ivf_build(ctypes.byref(args), _lib.stream_ptr())
    sizes = dict(ws=L.recnn_ivf_build_workspace_bytes(n, dim, nlist, 1500), centroids=nlist * dim * 4,
                 offsets=(nlist + 1) * 8, ids=n * 8, table=n * pitch * 4)
    if norms:
        sizes.update(cnorm=nlist * 4, norms=n * 4)
    check_windows(sizes, [(True, run)])


@pytest.mark.parametrize("k", [1, 17, 64])
@pytest.mark.parametrize("dim,metric", [(13, "COS"), (64, "L2"), (132, "IP")])
def test_workspace_bounds_search(dim, metric, k):
    x, q, index = _iid_index(metric, dim, n=5000, nlist=40)
    nq, nprobe = 40, 7
    qs = _dev(q)
    iv = index._ivf
    sets, flag = set_table(nq, 5000, dim), torch.zeros(1, dtype=torch.int32, device=DEV)

    def run(with_sets):
        def go(w, nbytes):
            sa = set_args(sets) if with_sets else (None, 0, None, 0, None)
            args = _lib.IvfSearchArgs(index._ivf_descriptor(iv), qs.data_ptr(), nq, nprobe, k, *sa, _ptr(w, "ids"),
                                      _ptr(w, "dist"), flag.data_ptr() if with_sets else None, _ptr(w, "ws"), nbytes)
            return L.recnn_ivf_search(ctypes.byref(args), _lib.stream_ptr())
        return go
    sizes = dict(ws=L.recnn_ivf_search_workspace_bytes(nq, iv["nlist"], nprobe, k), ids=nq * k * 8, dist=nq * k * 4)
    check_windows(sizes, [(True, run(False))])
    check_windows(sizes, [(True, run(True))], [flag], [flag])


# ---------------------------------------------------------------------------------------------------- scale
def test_scale_262144_items():
    n, dim, nlist = 262144, 128, 1024
    g = torch.Generator(device=DEV).manual_seed(0)
    table = torch.randn(n, dim, device=DEV, generator=g)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    index = ItemIndex(table, "L2").build_ivf(nlist, n_iter=10)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    table_bytes = n * dim * 4
    # the index (one list-ordered table + ids + norms) and the build's workspace (the sample, the sort buffers)
    assert peak < 3.2 * table_bytes, "peak %.1f MB over a %.1f MB table" % (peak / 2**20, table_bytes / 2**20)
    print("build peak %.1f MB over a %.1f MB table" % (peak / 2**20, table_bytes / 2**20))
    q = torch.randn(64, dim, device=DEV, generator=g)
    res = index.search(q, 10, search_param={"nprobe": 16})
    c, offsets, ids = _lists(index)
    probes = _device_probes(index, q, 16)
    xs, qs = _np(table), _np(q)
    want_i, want_d = V.probed_topk(qs, xs, "L2", probes, offsets, ids, 10)
    check_topk(_np(res.ids), _np(res.distances), want_i, want_d, qs, xs, "L2")
    exact = ItemIndex(table, "L2").search(q, 10).ids
    per_row, mean = recall_at_k(res.ids, exact)
    print("recall@10 at nprobe 16 over iid N(0, 1): %.3f" % mean)
