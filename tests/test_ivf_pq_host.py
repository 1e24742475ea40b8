"""The IVF_PQ oracle on the host (tests/_ivf_pq_oracle.py), the codeword sampling plan and the C ABI table."""
from __future__ import annotations

import ctypes

import numpy as np
import pytest

from recnn_b200 import _lib
from recnn_b200.data.db_con import ivf_pq_sample, ivf_sample
from tests import _ivf_oracle as V
from tests import _ivf_pq_oracle as P


def _small_index(metric, dim=12, m=4, n=300, nlist=6, seed=0):
    rng = np.random.default_rng(seed)
    table = rng.standard_normal((n, dim))
    c, offsets, ids = V.build(table, metric, nlist, n_iter=3)
    res = P.residuals(table, metric, c, offsets, ids)
    books = rng.standard_normal((m, 256, dim // m)) * 0.3
    codes, _ = P.encode(res, books)
    return table, c, offsets, ids, books, codes, P.item_lists(offsets, n, ids)


@pytest.mark.parametrize("metric", ["L2", "IP", "COS"])
def test_adc_keys_equal_the_reconstruction_values(metric):
    table, c, offsets, ids, books, codes, lists = _small_index(metric)
    q = np.random.default_rng(1).standard_normal((5, table.shape[1]))
    rec = P.reconstructions(c, books, codes, lists)
    want = P.reconstruction_values(q, rec, metric)
    got = P.adc_values(q, metric, c, books, codes, lists)
    np.testing.assert_allclose(got, want, rtol=1e-10, atol=1e-10)
    if metric == "L2":                                            # the squared distance to the reconstruction
        np.testing.assert_allclose(got[0], ((rec - q[0]) ** 2).sum(1), rtol=1e-10, atol=1e-10)


def test_encode_takes_the_nearest_codeword():
    rng = np.random.default_rng(2)
    books = rng.standard_normal((3, 256, 2))
    pick = rng.integers(0, 256, (50, 3))
    res = books[np.arange(3)[None, :], pick].reshape(50, 6) + 1e-6
    codes, d = P.encode(res, books)
    np.testing.assert_array_equal(codes, pick)
    assert (d.min(2) == d[np.arange(50)[:, None], np.arange(3)[None, :], codes]).all()


@pytest.mark.parametrize("metric", ["L2", "IP", "COS"])
def test_probed_topk_pads_orders_and_excludes(metric):
    table, c, offsets, ids, books, codes, lists = _small_index(metric, n=260, nlist=8)
    q = np.random.default_rng(3).standard_normal((4, table.shape[1]))
    values = P.adc_values(q, metric, c, books, codes, lists)
    probes = V.coarse(q, c, metric, 1)
    first = ids[offsets[probes[0, 0]]:offsets[probes[0, 0] + 1]]
    excl = [first[:3], None, [], first]
    got_i, got_d = P.probed_topk(values, metric, probes, offsets, ids, 64, exclude=excl)
    for r in range(4):
        l = probes[r, 0]
        members = set(ids[offsets[l]:offsets[l + 1]]) - set(np.asarray(excl[r] if excl[r] is not None else [],
                                                                        np.int64).tolist())
        filled = got_i[r][got_i[r] >= 0]
        assert set(filled) == members and len(filled) == len(members)
        assert np.isnan(got_d[r][len(filled):]).all()
        v = got_d[r][:len(filled)]
        assert (np.diff(v) >= 0).all() if metric == "L2" else (np.diff(v) <= 0).all()
        np.testing.assert_array_equal(v, values[r, filled])


def test_pq_sample_matches_the_oracle_plan():
    for n_sample, seed in [(1000, 0), (70000, 3), (256, 1)]:
        got = ivf_pq_sample(n_sample, seed).numpy()
        np.testing.assert_array_equal(got, P.pq_sample_plan(n_sample, seed))
        assert len(got) == 256 and len(set(got.tolist())) == 256 and got.max() < min(n_sample, 65536)
    s, _ = ivf_sample(100000, 16, 0, 256)                        # 4,096 training points
    assert ivf_pq_sample(len(s)).max() < 4096
    with pytest.raises(ValueError):
        ivf_pq_sample(255)


def test_ivf_pq_symbols_are_bound():
    L = _lib.lib()
    for name in ("recnn_ivf_pq_build_workspace_bytes", "recnn_ivf_pq_build", "recnn_ivf_pq_encode_workspace_bytes",
                 "recnn_ivf_pq_encode", "recnn_ivf_pq_search_workspace_bytes", "recnn_ivf_pq_search",
                 "recnn_sizeof_ivf_pq_index", "recnn_offsetof_ivf_pq_build_args", "recnn_offsetof_ivf_pq_encode_args",
                 "recnn_offsetof_ivf_pq_search_args"):
        assert name in _lib.SIGNATURES
        assert getattr(L, name) is not None
    with open(_lib._build.ROOT + "/include/recnn_b200.h") as fh:
        header = fh.read()
    for name in _lib.SIGNATURES:
        if "ivf_pq" in name:
            assert name + "(" in header, name


def test_argument_structs_match_the_library():
    L = _lib.lib()
    assert L.recnn_sizeof_ivf_pq_index() == ctypes.sizeof(_lib.IvfPqIndex)
    assert L.recnn_sizeof_ivf_pq_build_args() == ctypes.sizeof(_lib.IvfPqBuildArgs)
    assert L.recnn_sizeof_ivf_pq_encode_args() == ctypes.sizeof(_lib.IvfPqEncodeArgs)
    assert L.recnn_sizeof_ivf_pq_search_args() == ctypes.sizeof(_lib.IvfPqSearchArgs)
    for probe, cls, fields in ((L.recnn_offsetof_ivf_pq_build_args, _lib.IvfPqBuildArgs, _lib.IVF_PQ_BUILD_PROBE_FIELDS),
                               (L.recnn_offsetof_ivf_pq_encode_args, _lib.IvfPqEncodeArgs,
                                _lib.IVF_PQ_ENCODE_PROBE_FIELDS),
                               (L.recnn_offsetof_ivf_pq_search_args, _lib.IvfPqSearchArgs,
                                _lib.IVF_PQ_SEARCH_PROBE_FIELDS)):
        for i, f in enumerate(fields):
            assert probe(i) == getattr(cls, f).offset, f
        assert probe(len(fields)) == -1


def _index(**kw):
    a = dict(n_items=1000, dim=16, metric=_lib.METRIC_L2, nlist=8, m=4)
    a.update(kw)
    return _lib.IvfPqIndex(a["n_items"], a["dim"], a["metric"], a["nlist"], a["m"], 256, 256, 256, 256, 256, 256)


def test_calls_refuse_bad_arguments_before_device_work():
    L = _lib.lib()
    before = L.recnn_b200_launch_count()
    assert L.recnn_ivf_pq_search(None, None) == -1 and L.recnn_ivf_pq_build(None, None) == -1
    assert L.recnn_ivf_pq_encode(None, None) == -1
    ws = L.recnn_ivf_pq_search_workspace_bytes(4, 8, 4, 10, 4)

    def search(idx=None, **kw):
        a = _lib.IvfPqSearchArgs(idx or _index(), 256, 256, 256, 4, 4, 10, 4, 0, None, 0, None, 0, None, 256, 256,
                                 None, 256, ws)
        for k, v in kw.items():
            setattr(a, k, v)
        return L.recnn_ivf_pq_search(ctypes.byref(a), None)
    assert search(_index(m=3)) == -1                                        # m does not divide dim
    assert search(_index(m=65, dim=130)) == -1                              # m > 64
    assert search(_index(n_items=255)) == -1                                # fewer than 256 items
    assert search(_index(dim=516, m=4)) == -1                               # dim > 512
    assert search(refine=7) == -1                                           # refine * k > 64
    assert search(refine=-1) == -1
    assert search(nprobe=9) == -1                                           # nprobe > nlist
    assert search(refine=1, table=None) == -1                               # refine needs the table
    assert search(workspace_bytes=ws - 1) == -3                             # one byte short
    b = _lib.IvfPqBuildArgs(_index(), 256, 256, 500, 256, 256, 3, 0, 256,
                            L.recnn_ivf_pq_build_workspace_bytes(1000, 16, 8, 500, 4) - 1)
    assert L.recnn_ivf_pq_build(ctypes.byref(b), None) == -3
    b.n_sample = 200                                                        # fewer than 256 training points
    assert L.recnn_ivf_pq_build(ctypes.byref(b), None) == -1
    b.n_sample, b.n_iter = 500, -1
    assert L.recnn_ivf_pq_build(ctypes.byref(b), None) == -1
    e = _lib.IvfPqEncodeArgs(_index(), 256, 256, L.recnn_ivf_pq_encode_workspace_bytes(1000, 16) - 1)
    assert L.recnn_ivf_pq_encode(ctypes.byref(e), None) == -3
    e.index = _index(m=5)
    assert L.recnn_ivf_pq_encode(ctypes.byref(e), None) == -1
    assert L.recnn_b200_launch_count() == before


def test_workspace_queries_need_only_sizes():
    L = _lib.lib()
    a = L.recnn_ivf_pq_search_workspace_bytes(2048, 1024, 16, 10, 0)
    assert a > 0 and a == L.recnn_ivf_pq_search_workspace_bytes(2048, 1024, 16, 10, 1)
    assert L.recnn_ivf_pq_search_workspace_bytes(2048, 1024, 16, 10, 4) > a
    assert L.recnn_ivf_pq_search_workspace_bytes(2048, 8, 9, 10, 0) == 0    # nprobe > nlist
    b = L.recnn_ivf_pq_build_workspace_bytes(100000, 64, 256, 65536, 16)
    assert b > L.recnn_ivf_build_workspace_bytes(100000, 64, 256, 65536) + 65536 * 64 * 4
    assert L.recnn_ivf_pq_build_workspace_bytes(100000, 64, 256, 65536, 5) == 0   # m does not divide dim
    assert L.recnn_ivf_pq_build_workspace_bytes(255, 64, 4, 255, 16) == 0          # n_items < 256
    assert L.recnn_ivf_pq_encode_workspace_bytes(10**6, 256) >= 65536 * 256 * 4
