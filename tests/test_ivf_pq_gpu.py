"""IVF_PQ on the device (recnn_ivf_pq_build / _encode / _search behind ItemIndex.build_ivf(..., m=M) and search) against
the float64 oracle of tests/_ivf_pq_oracle.py and against IVF_FLAT over the same lists."""
from __future__ import annotations

import ctypes
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from recnn_b200 import _lib
from recnn_b200.data import ItemIndex, ItemSets, MilvusConnection
from recnn_b200.utils.metrics import recall_at_k
from tests import _ivf_oracle as V
from tests import _ivf_pq_oracle as P
from tests.test_ivf_gpu import _dev, _device_probes, _lists, _np, _tol, _values64, check_topk
from tests.test_workspace_bounds_serving_gpu import _ptr, check_windows, set_args, set_table

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
L = _lib.lib()
METRICS = ["L2", "IP", "COS"]
DIM_M = [(13, 13), (64, 16), (132, 12)]     # dsub 1, 4 and 11


def _indexes(metric, dim, m, n=3000, nlist=32, seed=0):
    """table, queries, the IVF_FLAT index and the IVF_PQ index built with the same arguments"""
    rng = np.random.default_rng(seed + dim)
    x = rng.standard_normal((n, dim)).astype(np.float32)
    q = rng.standard_normal((40, dim)).astype(np.float32)
    flat = ItemIndex(_dev(x), metric).build_ivf(nlist, n_iter=5, seed=seed)
    pq = ItemIndex(_dev(x), metric).build_ivf(nlist, n_iter=5, seed=seed, m=m)
    return x, q, flat, pq


def _pq_host(index):
    """centroids, offsets, ids, codebooks, codes by item id, the list of each item (numpy)"""
    c, offsets, ids = _lists(index)
    books, codes = index.pq
    by_item = np.empty((index.n_items, codes.shape[1]), np.int64)
    by_item[ids] = _np(codes).astype(np.int64)
    return c, offsets, ids, _np(books).astype(np.float64), by_item, P.item_lists(offsets, index.n_items, ids)


def _check_adc(got, q, metric, index, probes, k, exclude=None):
    """the device's ADC top-k against the oracle's over the device's codebooks, codes and probes"""
    c, offsets, ids, books, codes, lists = _pq_host(index)
    values = P.adc_values(q, metric, c, books, codes, lists)
    want_i, want_d = P.probed_topk(values, metric, probes, offsets, ids, k, exclude=exclude)
    rec = P.reconstructions(c, books, codes, lists)
    # COS is the IP form on the unit query against the reconstruction
    qq, mm = (V._unit(np.asarray(q, np.float64)), "IP") if metric == "COS" else (q, metric)
    check_topk(_np(got.ids), _np(got.distances), want_i, want_d, qq, rec, mm)


def _long_lists(metric, dim, m, seed=0):
    """6,000 items in 2 lists: about 3,000 items a list, so a work unit streams about 12 chunks of 256 codes through
    both buffers and its tail, and each of the S = 32 threads of a query (m <= 16) sees about 94 items of a list, more
    than either register list (16 or 64 entries) holds"""
    x, q, flat, pq = _indexes(metric, dim, m, n=6000, nlist=2, seed=seed)
    lens = np.diff(_np(pq.ivf.list_offsets))
    assert lens.min() >= 3 * 256 and lens.min() // 32 > 64, lens
    return x, q, flat, pq


# ---------------------------------------------------------------------------------------------------- build
@pytest.mark.parametrize("dim,m", DIM_M)
@pytest.mark.parametrize("metric", METRICS)
def test_coarse_lists_equal_ivf_flat_and_builds_repeat(metric, dim, m):
    x, q, flat, pq = _indexes(metric, dim, m)
    for k in ("centroids", "centroid_norms", "list_offsets", "list_ids"):
        a, b = flat._ivf[k], pq._ivf[k]
        assert (a is None and b is None) or torch.equal(a, b), k
    again = ItemIndex(_dev(x), metric).build_ivf(32, n_iter=5, seed=0, m=m)
    for k in ("centroids", "list_offsets", "list_ids", "codebooks", "codes"):
        assert torch.equal(pq._ivf[k], again._ivf[k]), k
    books, codes = pq.pq
    assert books.shape == (m, 256, dim // m) and codes.shape == (len(x), m) and codes.dtype == torch.uint8
    assert flat.pq is None and pq.ivf is not None
    assert bool((pq._ivf["codes"][:, m:] == 0).all())                   # the 16-byte row padding


@pytest.mark.parametrize("dim,m", DIM_M)
@pytest.mark.parametrize("metric", METRICS)
def test_every_code_is_an_argmin(metric, dim, m):
    x, q, flat, pq = _indexes(metric, dim, m)
    c, offsets, ids, books, codes, lists = _pq_host(pq)
    res = P.residuals(x, metric, c, offsets, ids)
    _, d = P.encode(res, books)                                          # [n, m, 256]
    chosen = np.take_along_axis(d, codes[:, :, None], 2)[:, :, 0]
    best = d.min(2)
    slack = chosen - best
    bar = 1e-5 * (1.0 + d.max())
    assert (slack <= bar).all(), "a code misses the argmin by %g" % slack.max()
    print("codes not the float64 argmin (fp32 near-ties): %d of %d" % (int((slack > 0).sum()), slack.size))


def test_codebooks_recover_subspace_blobs():
    # one list, and per subspace eight well separated blobs: every blob centre (relative to the centroid) gets a
    # codeword, and every item's codeword is its blob's
    rng = np.random.default_rng(4)
    n, dim, m = 2048, 16, 4
    centres = rng.standard_normal((m, 8, dim // m)) * 5.0
    labels = rng.integers(0, 8, (n, m))
    x = np.concatenate([centres[j][labels[:, j]] for j in range(m)], axis=1) + 0.01 * rng.standard_normal((n, dim))
    index = ItemIndex(_dev(x), "L2").build_ivf(1, n_iter=10, m=m)
    c, offsets, ids, books, codes, lists = _pq_host(index)
    for j in range(m):
        cj = centres[j] - c[0].reshape(m, -1)[j]
        gap = np.linalg.norm(cj[:, None, :] - books[j][None], axis=2).min(1)
        assert (gap < 0.05).all(), (j, gap)
        picked = books[j][codes[:, j]]
        np.testing.assert_allclose(picked, cj[labels[:, j]], atol=0.05)


def test_build_refuses_bad_arguments():
    index = ItemIndex(torch.randn(300, 12, device=DEV), "L2")
    for kw in (dict(m=5), dict(m=0), dict(m=24), dict(m=4, max_points_per_centroid=10)):
        with pytest.raises(ValueError):
            index.build_ivf(4, **kw)
    with pytest.raises(ValueError):
        ItemIndex(torch.randn(200, 12, device=DEV), "L2").build_ivf(4, m=4)        # n_items < 256
    with pytest.raises(ValueError):
        ItemIndex(torch.randn(300, 130, device=DEV), "L2").build_ivf(4, m=65)
    assert index.ivf is None and index.pq is None


# ---------------------------------------------------------------------------------------------------- search
@pytest.mark.parametrize("k", [1, 10, 64])
@pytest.mark.parametrize("nprobe", [1, 4, 16])
@pytest.mark.parametrize("dim,m", DIM_M)
@pytest.mark.parametrize("metric", METRICS)
def test_adc_search_matches_oracle(metric, dim, m, nprobe, k):
    x, q, flat, pq = _indexes(metric, dim, m)
    got = pq.search(_dev(q), k, search_param={"nprobe": nprobe})
    _check_adc(got, q, metric, pq, _device_probes(pq, _dev(q), nprobe), k)


@pytest.mark.parametrize("k", [10, 64])
@pytest.mark.parametrize("nprobe", [1, 2])
@pytest.mark.parametrize("dim,m", DIM_M)
@pytest.mark.parametrize("metric", METRICS)
def test_adc_search_matches_oracle_on_long_lists(metric, dim, m, nprobe, k):
    x, q, flat, pq = _long_lists(metric, dim, m)
    got = pq.search(_dev(q), k, search_param={"nprobe": nprobe})
    _check_adc(got, q, metric, pq, _device_probes(pq, _dev(q), nprobe), k)


@pytest.mark.parametrize("k,refine", [(8, 2), (10, 4)])
@pytest.mark.parametrize("dim,m", DIM_M)
@pytest.mark.parametrize("metric", METRICS)
def test_refine_on_long_lists_equals_ivf_flat_over_the_candidates(metric, dim, m, k, refine):
    # k' = 16 and 40 cannot cover a 3,000-item list, so the bit-level check runs IVF_FLAT over exactly the device's
    # k' ADC candidates (every other item excluded): refine must return that search's ids and distances, bit for bit
    x, q, flat, pq = _long_lists(metric, dim, m)
    qs, kp = _dev(q), k * refine
    cand = pq.search(qs, kp, search_param={"nprobe": 2})            # the same k' lists the refine pass merges
    _check_adc(cand, q, metric, pq, _device_probes(pq, qs, 2), kp)
    got = pq.search(qs, k, search_param={"nprobe": 2, "refine": refine})
    others = [np.setdiff1d(np.arange(len(x)), row) for row in _np(cand.ids)]
    want = flat.search(qs, k, search_param={"nprobe": 2}, exclude=ItemSets.from_lists(others, device=DEV))
    assert torch.equal(got.ids, want.ids) and torch.equal(got.distances, want.distances)


@pytest.mark.parametrize("dim,m", DIM_M)
@pytest.mark.parametrize("metric", METRICS)
def test_full_coverage_refine_equals_ivf_flat(metric, dim, m):
    rng = np.random.default_rng(dim)
    x = _dev(rng.standard_normal((512, dim)))
    q = _dev(rng.standard_normal((64, dim)))
    flat = ItemIndex(x, metric).build_ivf(64, n_iter=4)
    pq = ItemIndex(x, metric).build_ivf(64, n_iter=4, m=m)
    k, refine, nprobe = 8, 8, 2
    want = flat.search(q, k, search_param={"nprobe": nprobe})
    got = pq.search(q, k, search_param={"nprobe": nprobe, "refine": refine})
    c, offsets, ids = _lists(pq)
    probes = _device_probes(pq, q, nprobe)
    union = np.array([sum(offsets[l + 1] - offsets[l] for l in probes[r]) for r in range(len(probes))])
    covered = torch.from_numpy(union <= k * refine).to(DEV)
    assert covered.float().mean() > 0.5, union
    assert torch.equal(got.ids[covered], want.ids[covered])
    assert torch.equal(got.distances[covered], want.distances[covered])


@pytest.mark.parametrize("dim,m", DIM_M)
@pytest.mark.parametrize("metric", METRICS)
def test_refine_returns_exact_distances(metric, dim, m):
    x, q, flat, pq = _indexes(metric, dim, m)
    got = pq.search(_dev(q), 10, search_param={"nprobe": 8, "refine": 2})
    gi, gd = _np(got.ids), _np(got.distances)
    assert (gi >= 0).all()
    np.testing.assert_allclose(gd, _values64(q, x, gi, metric), atol=_tol(q, x, metric), rtol=0)
    c, offsets, ids = _lists(pq)
    probes = _device_probes(pq, _dev(q), 8)
    for r in range(len(q)):
        union = set(np.concatenate([ids[offsets[l]:offsets[l + 1]] for l in probes[r]]).tolist())
        assert set(gi[r].tolist()) <= union
        assert len(set(gi[r].tolist())) == 10
    order = gd if metric == "L2" else -gd
    assert (np.diff(order, axis=1) >= -_tol(q, x, metric)).all()
    # refine can only help: the exact top-k over the probed lists is at least as well recalled as ADC's
    exact = flat.search(_dev(q), 10, search_param={"nprobe": 8}).ids
    adc = pq.search(_dev(q), 10, search_param={"nprobe": 8}).ids
    print("recall@10 vs IVF_FLAT: adc %.3f, refine 2 %.3f" % (recall_at_k(adc, exact)[1],
                                                              recall_at_k(got.ids, exact)[1]))


@pytest.mark.parametrize("long_lists", [False, True])
@pytest.mark.parametrize("k,refine", [(10, 0), (17, 0), (17, 2)])
@pytest.mark.parametrize("metric", METRICS)
def test_batch_invariance(metric, k, refine, long_lists):
    # k' = 10 runs the 16-entry register lists, 17 and 34 the 64-entry ones; long lists stream many chunks per unit
    x, q, flat, pq = _long_lists(metric, 64, 16) if long_lists else _indexes(metric, 64, 16)
    qs = _dev(q)
    sp = {"nprobe": 2 if long_lists else 8, "refine": refine}
    full = pq.search(qs, k, search_param=sp)
    perm = torch.randperm(len(q), generator=torch.Generator().manual_seed(0)).to(DEV)
    shuffled = pq.search(qs[perm], k, search_param=sp)
    assert torch.equal(shuffled.ids, full.ids[perm]) and torch.equal(shuffled.distances, full.distances[perm])
    big = torch.cat([qs, _dev(np.random.default_rng(1).standard_normal((3000, 64)))])
    many = pq.search(big, k, search_param=sp)
    assert torch.equal(many.ids[:len(q)], full.ids) and torch.equal(many.distances[:len(q)], full.distances)
    for r in (0, 7, len(q) - 1):
        one = pq.search(qs[r:r + 1], k, search_param=sp)
        assert torch.equal(one.ids[0], full.ids[r]) and torch.equal(one.distances[0], full.distances[r])


def test_search_param_checks():
    x, q, flat, pq = _indexes("L2", 16, 4, nlist=20)
    qs = _dev(q)
    assert torch.equal(pq.search(qs, 5).ids, pq.search(qs, 5, search_param={"nprobe": 16, "refine": 0}).ids)
    for bad in ({"nprobe": 0}, {"nprobe": 21}, {"refine": -1}, {"refine": 13}, {"nprobe": 4, "ef": 3}):
        with pytest.raises(ValueError):
            pq.search(qs, 5, search_param=bad)
    pq.search(qs, 5, search_param={"refine": 12})                             # 12 * 5 <= 64
    with pytest.raises(ValueError):
        flat.search(qs, 5, search_param={"nprobe": 4, "refine": 1})           # refine on IVF_FLAT
    target = torch.arange(len(q), device=DEV)
    assert torch.equal(pq.rank(qs, target), ItemIndex(_dev(x), "L2").rank(qs, target))
    assert pq.search(qs[:0], 5).ids.shape == (0, 5)


@pytest.mark.parametrize("refine", [0, 3])
@pytest.mark.parametrize("metric", METRICS)
def test_exclusion(metric, refine):
    x, q, flat, pq = _indexes(metric, 64, 16, n=2000, nlist=64)
    c, offsets, ids = _lists(pq)
    probes = _device_probes(pq, _dev(q), 2)
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
    res = pq.search(_dev(q), 10, search_param={"nprobe": 2, "refine": refine}, exclude=ex)
    got_i, got_d = _np(res.ids), _np(res.distances)
    for r in range(len(q)):
        assert not set(got_i[r][got_i[r] >= 0]) & set(sets[r].tolist())
    if refine == 0:
        _check_adc(res, q, metric, pq, probes, 10, exclude=sets)
    else:
        ok = got_i >= 0
        np.testing.assert_allclose(got_d[ok], _values64(q, x, got_i, metric)[ok], atol=_tol(q, x, metric), rtol=0)
    pad = got_i == -1
    assert pad[0].any() and (pad[0].sum() == 10 - (len(np.concatenate([ids[offsets[l]:offsets[l + 1]]
                                                                         for l in probes[0]])) - len(sets[0])))
    assert (got_d[pad] == (np.finfo(np.float32).max if metric == "L2" else -np.finfo(np.float32).max)).all()
    with pytest.raises(IndexError):
        pq.search(_dev(q[:2]), 5, exclude=ItemSets.from_lists([[0, len(x)], [1]], device=DEV))
    bad = ItemSets.from_lists([[3, 1]], device=DEV)
    bad.ids = torch.tensor([3, 1], device=DEV)                     # descending: malformed
    with pytest.raises(ValueError):
        pq.search(_dev(q[:1]), 5, exclude=bad)


# ---------------------------------------------------------------------------------------------------- persistence
@pytest.mark.parametrize("metric", METRICS)
def test_state_round_trip(metric):
    x, q, flat, pq = _indexes(metric, 132, 12)
    state = pq.ivf_state()
    assert state["params"]["m"] == 12 and tuple(state["codebooks"].shape) == (12, 256, 11)
    fresh = ItemIndex(_dev(x), metric).load_ivf(state)
    for k in ("centroids", "centroid_norms", "list_offsets", "list_ids", "codebooks", "codes"):
        a, b = pq._ivf[k], fresh._ivf[k]
        assert (a is None and b is None) or torch.equal(a, b), k
    for sp in ({"nprobe": 4}, {"nprobe": 4, "refine": 2}):
        want = pq.search(_dev(q), 10, search_param=sp)
        got = fresh.search(_dev(q), 10, search_param=sp)
        assert torch.equal(want.ids, got.ids) and torch.equal(want.distances, got.distances)
    assert fresh.ivf_state()["params"] == state["params"]
    assert "codebooks" not in flat.ivf_state()


def test_load_refuses_corrupted_state():
    x, q, flat, pq = _indexes("L2", 16, 4)
    good = pq.ivf_state()

    def with_(**kw):
        s = dict(good)
        s.update(kw)
        return s
    no_books = dict(good)
    del no_books["codebooks"]
    swapped = good["list_ids"].clone()
    swapped[0] = good["list_ids"][1]
    for s in (no_books, with_(codebooks=good["codebooks"][:3]), with_(codebooks=good["codebooks"][:, :255]),
              with_(codebooks=good["codebooks"].to(torch.int64)), with_(params=dict(good["params"], m=5)),
              with_(params=dict(good["params"], m="4")), with_(list_ids=swapped), with_(metric="IP")):
        with pytest.raises(ValueError):
            ItemIndex(_dev(x), "L2").load_ivf(s)


def test_milvus_connection_builds_ivf_pq():
    x = torch.randn(600, 16, device=DEV)
    conn = MilvusConnection(x, param={"index_type": "IVF_PQ", "nlist": 10, "m": 8, "nbits": 8})
    assert conn.pq is not None and conn.pq[0].shape == (8, 256, 2) and conn.ivf.centroids.shape == (10, 16)
    assert MilvusConnection(x, param={"index_type": "IVF_PQ", "nlist": 10, "m": 4}).pq[1].shape == (600, 4)
    for bad in ({"index_type": "IVF_PQ", "nlist": 10}, {"index_type": "IVF_PQ", "nlist": 10, "m": 8, "nbits": 4},
                {"index_type": "HNSW"}):
        with pytest.raises(ValueError):
            MilvusConnection(x, param=bad)


# ---------------------------------------------------------------------------------------------------- workspace contract
def _pq_buffers(n, dim, nlist, m, norms):
    pitch = (m + 15) // 16 * 16
    sizes = dict(centroids=nlist * dim * 4, offsets=(nlist + 1) * 8, ids=n * 8, books=256 * dim * 4, codes=n * pitch)
    if norms:
        sizes["cnorm"] = nlist * 4
    return sizes


def _pq_desc(w, n, dim, metric, nlist, m, norms):
    return _lib.ivf_pq_index(n, dim, metric, nlist, m, w["centroids"], w["cnorm"] if norms else None, w["offsets"],
                             w["ids"], w["books"], w["codes"])


@pytest.mark.parametrize("dim,m,metric", [(13, 13, _lib.METRIC_COS), (64, 16, _lib.METRIC_L2),
                                          (132, 33, _lib.METRIC_IP)])
def test_workspace_bounds_build_and_encode(dim, m, metric):
    n, nlist = 3001, 24
    torch.manual_seed(dim)
    table = torch.randn(n, dim, device=DEV)
    sample = torch.randperm(n, device=DEV)[:1500].contiguous()
    init = torch.randperm(1500, device=DEV)[:nlist].contiguous()
    pq_init = torch.randperm(1500, device=DEV)[:256].contiguous()
    norms = metric != _lib.METRIC_IP

    def build(w, nbytes):
        args = _lib.IvfPqBuildArgs(_pq_desc(w, n, dim, metric, nlist, m, norms), table.data_ptr(), sample.data_ptr(),
                                   1500, init.data_ptr(), pq_init.data_ptr(), 3, 0, _ptr(w, "ws"), nbytes)
        return L.recnn_ivf_pq_build(ctypes.byref(args), _lib.stream_ptr())
    sizes = dict(ws=L.recnn_ivf_pq_build_workspace_bytes(n, dim, nlist, 1500, m), **_pq_buffers(n, dim, nlist, m, norms))
    check_windows(sizes, [(True, build)])

    # encode over a built index's lists and codebooks
    index = ItemIndex(table, ["L2", "IP", "COS"][metric]).build_ivf(nlist, n_iter=3, m=m)
    iv = index._ivf
    codes = torch.empty_like(iv["codes"])

    def encode(w, nbytes):
        desc = _lib.ivf_pq_index(n, dim, metric, nlist, m, iv["centroids"], iv["centroid_norms"], iv["list_offsets"],
                                 iv["list_ids"], iv["codebooks"], w["codes"])
        args = _lib.IvfPqEncodeArgs(desc, table.data_ptr(), _ptr(w, "ws"), nbytes)
        return L.recnn_ivf_pq_encode(ctypes.byref(args), _lib.stream_ptr())
    check_windows(dict(ws=L.recnn_ivf_pq_encode_workspace_bytes(n, dim), codes=codes.numel()), [(True, encode)])


@pytest.mark.parametrize("k,refine", [(1, 0), (17, 3), (64, 1)])
@pytest.mark.parametrize("dim,m,metric", [(13, 13, "COS"), (64, 16, "L2"), (132, 33, "IP")])
def test_workspace_bounds_search(dim, m, metric, k, refine):
    x, q, flat, pq = _indexes(metric, dim, m, n=5000, nlist=40)
    nq, nprobe = 40, 7
    qs = _dev(q)
    iv = pq._ivf
    sets, flag = set_table(nq, 5000, dim), torch.zeros(1, dtype=torch.int32, device=DEV)

    def run(with_sets):
        def go(w, nbytes):
            sa = set_args(sets) if with_sets else (None, 0, None, 0, None)
            args = _lib.IvfPqSearchArgs(pq._pq_descriptor(iv), pq.table.data_ptr(), _lib.ptr(pq.norms), qs.data_ptr(),
                                        nq, nprobe, k, refine, 0, *sa, _ptr(w, "ids"), _ptr(w, "dist"),
                                        flag.data_ptr() if with_sets else None, _ptr(w, "ws"), nbytes)
            return L.recnn_ivf_pq_search(ctypes.byref(args), _lib.stream_ptr())
        return go
    sizes = dict(ws=L.recnn_ivf_pq_search_workspace_bytes(nq, iv["nlist"], nprobe, k, refine), ids=nq * k * 8,
                 dist=nq * k * 4)
    check_windows(sizes, [(True, run(False))])
    check_windows(sizes, [(True, run(True))], [flag], [flag])


# ---------------------------------------------------------------------------------------------------- scale
def test_scale_262144_items():
    n, dim, nlist, m = 262144, 128, 1024, 32
    g = torch.Generator(device=DEV).manual_seed(0)
    table = torch.randn(n, dim, device=DEV, generator=g)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    index = ItemIndex(table, "L2").build_ivf(nlist, n_iter=10, m=m)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    table_bytes = n * dim * 4
    # the build's workspace: the IVF_FLAT coarse build's (the sample, the sort buffers), the training residuals and
    # one encode slab; the index itself is small
    assert peak < 2.0 * table_bytes, "peak %.1f MB over a %.1f MB table" % (peak / 2**20, table_bytes / 2**20)
    nbytes = sum(t.numel() * t.element_size() for t in index._ivf.values() if torch.is_tensor(t))
    bound = n * (m + 8) + nlist * dim * 4 + 256 * dim * 4 + 2**20
    assert nbytes <= bound, (nbytes, bound)
    print("build peak %.1f MB over a %.1f MB table; index %.1f MB" % (peak / 2**20, table_bytes / 2**20,
                                                                       nbytes / 2**20))
    q = torch.randn(64, dim, device=DEV, generator=g)
    exact = ItemIndex(table, "L2").search(q, 10).ids
    res = index.search(q, 10, search_param={"nprobe": 16, "refine": 4})
    np.testing.assert_allclose(_np(res.distances), _values64(_np(q), _np(table), _np(res.ids), "L2"),
                               atol=_tol(_np(q), _np(table), "L2"), rtol=0)
    adc = index.search(q, 10, search_param={"nprobe": 16})
    # the ADC result over lists of about 256 items (nlist 1,024), several chunks for the longest, against the oracle
    _check_adc(SimpleNamespace(ids=adc.ids[:16], distances=adc.distances[:16]), _np(q[:16]), "L2", index,
               _device_probes(index, q[:16], 16), 10)
    print("recall@10 over iid N(0, 1) at nprobe 16: refine 4 %.3f, adc %.3f"
          % (recall_at_k(res.ids, exact)[1], recall_at_k(adc.ids, exact)[1]))
