"""The IVF_FLAT oracle on the host (tests/_ivf_oracle.py), the sampling plan, recall_at_k and the C ABI table."""
from __future__ import annotations

import ctypes

import numpy as np
import pytest
import torch

from oracle import recnn_oracle as O
from recnn_b200 import _lib
from recnn_b200.data.db_con import ivf_sample
from recnn_b200.utils.metrics import recall_at_k
from tests import _ivf_oracle as V


def _first_seed_covering(labels, nlist, n_blobs, start=0):
    """a seed whose init takes one point of every blob (Lloyd from there converges to the blobs)"""
    for seed in range(start, start + 200):
        _, init = V.sample_plan(len(labels), nlist, seed)
        if len(set(labels[init])) == n_blobs:
            return seed
    raise AssertionError("no covering seed")


@pytest.mark.parametrize("metric", ["L2", "IP", "COS"])
def test_oracle_recovers_separated_blobs(metric):
    rng = np.random.default_rng(3)
    centers = rng.standard_normal((6, 16))
    centers = 20.0 * centers / np.linalg.norm(centers, axis=1, keepdims=True)
    x, labels = V.blobs(50, centers, 0.3, seed=4)
    seed = _first_seed_covering(labels, 6, 6)
    c, offsets, ids = V.build(x, metric, 6, n_iter=10, seed=seed)
    assert offsets[0] == 0 and offsets[-1] == len(x)
    got = sorted(tuple(ids[offsets[l]:offsets[l + 1]]) for l in range(6))
    want = sorted(tuple(np.nonzero(labels == b)[0]) for b in range(6))
    assert got == want
    for l in range(6):                                          # each centroid sits on its blob's mean
        members = x[ids[offsets[l]:offsets[l + 1]]]
        mean = members.mean(0) if metric != "COS" else V._unit((members / np.linalg.norm(members, axis=1,
                                                                                          keepdims=True)).mean(0)[None])[0]
        np.testing.assert_allclose(c[l], mean, atol=1e-9)


def test_empty_cluster_split_fires_and_is_deterministic():
    # two identical initial centroids: the second gets no members (ties go to the smaller id) and is split off the
    # largest list
    x = np.array([[0.0, 0.0], [0.1, 0.0], [0.0, 0.1], [5.0, 5.0], [5.1, 5.0], [9.0, 0.0], [9.0, 0.2], [9.1, 0.1],
                  [9.2, 0.0]])
    init = x[[0, 0, 3]]
    c = init.copy()
    a = V.assign(x, c)
    counts = np.bincount(a, minlength=3).astype(np.float64)
    assert counts[1] == 0
    for l in np.nonzero(counts)[0]:
        c[l] = x[a == l].mean(0)
    donor = int(np.argmax(counts))
    v = c[donor].copy()
    pairs = V.split_empty(c, counts)
    assert pairs == [(1, donor)]
    np.testing.assert_array_equal(c[1], v * np.array([1 + V.EPS, 1 - V.EPS]))
    np.testing.assert_array_equal(c[donor], v * np.array([1 - V.EPS, 1 + V.EPS]))
    assert counts[1] == counts[donor] == 3.0
    r1 = V.lloyd(x, init, 5, False)
    r2 = V.lloyd(x, init, 5, False)
    np.testing.assert_array_equal(r1, r2)
    assert len(set(V.assign(x, r1))) == 3                   # the split list found members


def test_split_ties_go_to_the_smaller_donor():
    c = np.arange(8, dtype=np.float64).reshape(4, 2) + 1.0
    counts = np.array([0.0, 4.0, 4.0, 0.0])
    assert V.split_empty(c, counts) == [(0, 1), (3, 2)]
    np.testing.assert_array_equal(counts, [2.0, 2.0, 2.0, 2.0])


@pytest.mark.parametrize("metric", ["L2", "IP", "COS"])
def test_full_probe_equals_exact_search(metric):
    rng = np.random.default_rng(7)
    table, queries = rng.standard_normal((400, 12)), rng.standard_normal((9, 12))
    c, offsets, ids = V.build(table, metric, 8, n_iter=4)
    probes = V.coarse(queries, c, metric, 8)
    got_i, got_d = V.probed_topk(queries, table, metric, probes, offsets, ids, 10)
    want_i, want_d = O.retrieve_topk(queries, table, 10, metric)
    np.testing.assert_array_equal(got_i, want_i)
    np.testing.assert_allclose(got_d, want_d, rtol=1e-12, atol=1e-12)


def test_probed_topk_pads_short_unions_and_excludes():
    rng = np.random.default_rng(8)
    table, queries = rng.standard_normal((60, 5)), rng.standard_normal((3, 5))
    c, offsets, ids = V.build(table, "L2", 6, n_iter=3)
    probes = V.coarse(queries, c, "L2", 1)
    excl = [ids[offsets[probes[0, 0]]:offsets[probes[0, 0] + 1]][:2], None, []]
    got_i, got_d = V.probed_topk(queries, table, "L2", probes, offsets, ids, 64, exclude=excl)
    for r in range(3):
        l = probes[r, 0]
        members = set(ids[offsets[l]:offsets[l + 1]]) - set(excl[r] if excl[r] is not None else [])
        filled = got_i[r][got_i[r] >= 0]
        assert set(filled) == members and len(filled) == len(members)
        assert np.isnan(got_d[r][len(filled):]).all()


def test_sample_plan_matches_the_package():
    for n, nlist, mppc, seed in [(1000, 10, 256, 0), (1000, 10, 7, 3), (5, 5, 1, 1)]:
        s, i = ivf_sample(n, nlist, seed, mppc)
        vs, vi = V.sample_plan(n, nlist, seed, mppc)
        np.testing.assert_array_equal(s.numpy(), vs)
        np.testing.assert_array_equal(i.numpy(), vi)
        assert len(s) == min(n, nlist * mppc) and len(set(s.tolist())) == len(s)
        assert len(i) == nlist and int(i.max()) < len(s)
    s, _ = ivf_sample(1000, 10, 0, 256)
    np.testing.assert_array_equal(s.numpy(), np.arange(1000))    # small tables train on every item


def test_recall_at_k():
    exact = torch.tensor([[1, 2, 3, 4], [5, 6, -1, -1], [-1, -1, -1, -1]])
    approx = torch.tensor([[4, 9, 1, 8], [6, 5, 7, -1], [1, 2, 3, 4]])
    per_row, mean = recall_at_k(approx, exact)
    assert per_row[:2].tolist() == [0.5, 1.0] and np.isnan(float(per_row[2]))
    assert mean == 0.75
    with pytest.raises(ValueError):
        recall_at_k(torch.zeros(3, 2), exact)
    with pytest.raises(ValueError):
        recall_at_k(approx[:2], exact)
    assert np.isnan(recall_at_k(torch.full((1, 2), -1), torch.full((1, 2), -1))[1])


def test_ivf_symbols_are_bound():
    for name in ("recnn_ivf_build_workspace_bytes", "recnn_ivf_build", "recnn_ivf_list_table",
                 "recnn_ivf_search_workspace_bytes", "recnn_ivf_search"):
        assert name in _lib.SIGNATURES


def test_argument_structs_match_the_library():
    L = _lib.lib()
    assert L.recnn_sizeof_ivf_index() == ctypes.sizeof(_lib.IvfIndex)
    assert L.recnn_sizeof_ivf_build_args() == ctypes.sizeof(_lib.IvfBuildArgs)
    assert L.recnn_sizeof_ivf_search_args() == ctypes.sizeof(_lib.IvfSearchArgs)
    for i, f in enumerate(_lib.IVF_BUILD_PROBE_FIELDS):
        assert L.recnn_offsetof_ivf_build_args(i) == getattr(_lib.IvfBuildArgs, f).offset, f
    for i, f in enumerate(_lib.IVF_SEARCH_PROBE_FIELDS):
        assert L.recnn_offsetof_ivf_search_args(i) == getattr(_lib.IvfSearchArgs, f).offset, f
    assert L.recnn_offsetof_ivf_search_args(len(_lib.IVF_SEARCH_PROBE_FIELDS)) == -1


def test_calls_refuse_bad_arguments_before_device_work():
    L = _lib.lib()
    before = L.recnn_b200_launch_count()
    assert L.recnn_ivf_search(None, None) == -1 and L.recnn_ivf_build(None, None) == -1
    idx = _lib.IvfIndex(1000, 16, _lib.METRIC_L2, 8, 0, 256, 256, 256, 256, 256, 256)
    a = _lib.IvfSearchArgs(idx, 256, 4, 9, 10, None, 0, None, 0, None, 256, 256, None, 256, 1 << 30)
    assert L.recnn_ivf_search(ctypes.byref(a), None) == -1                  # nprobe > nlist
    a.nprobe, a.k = 4, 65
    assert L.recnn_ivf_search(ctypes.byref(a), None) == -1                  # k > 64
    a.k, a.workspace_bytes = 10, L.recnn_ivf_search_workspace_bytes(4, 8, 4, 10) - 1
    assert L.recnn_ivf_search(ctypes.byref(a), None) == -3                  # one byte short
    b = _lib.IvfBuildArgs(idx, 256, 256, 500, 256, 3, 0, 256, L.recnn_ivf_build_workspace_bytes(1000, 16, 8, 500) - 1)
    assert L.recnn_ivf_build(ctypes.byref(b), None) == -3
    b.n_iter = -1
    assert L.recnn_ivf_build(ctypes.byref(b), None) == -1
    assert L.recnn_b200_launch_count() == before


def test_workspace_queries_need_only_sizes():
    L = _lib.lib()
    a = L.recnn_ivf_search_workspace_bytes(2048, 1024, 16, 10)
    assert a > 0 and a == L.recnn_ivf_search_workspace_bytes(2048, 1024, 16, 10)
    assert L.recnn_ivf_search_workspace_bytes(2048, 1024, 16, 64) > a
    assert L.recnn_ivf_search_workspace_bytes(2048, 8, 9, 10) == 0          # nprobe > nlist
    b = L.recnn_ivf_build_workspace_bytes(100000, 64, 256, 65536)
    assert b > 100000 * 64 * 0 and b > 65536 * 64 * 4
    assert L.recnn_ivf_build_workspace_bytes(100, 64, 256, 100) == 0         # nlist > n_sample
