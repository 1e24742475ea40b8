"""The scipy.spatial.distance metrics of ItemIndex on the host: the fp32 replay (tests/_metric_oracle.py) against
scipy's cdist and against the demo's ranking (examples/streamlit_demo.py:207-230: sorted(items, key=metric)[:k]), the
conventions where scipy gives NaN, the refusals of the Python and C layers, and the header's metric codes."""
from __future__ import annotations

import ctypes
import os
import re

import numpy as np
import pytest
import torch

from recnn_b200 import _lib
from recnn_b200.data.db_con import ItemIndex
from tests import _metric_oracle as M

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
U = 2.0 ** -24


def _scipy_fn(name, p=None):
    from scipy.spatial import distance
    f = getattr(distance, name)
    return (lambda u, v: f(u, v, p=2 if p is None else p)) if name == "minkowski" else f


@pytest.mark.parametrize("name", M.SCIPY_NAMES)
def test_replay_matches_cdist_on_small_ints(name):
    """Entries in {-1, 0, 1}: every fp32 step of cityblock, chebyshev, canberra (terms 0 or 1), braycurtis (one
    division of integers) and euclidean (the sqrt of an integer) is exact or one correct rounding of scipy's value."""
    rng = np.random.default_rng(11)
    table, q = M.small_ints(rng, (300, 16), -1, 1), M.small_ints(rng, (6, 16), -1, 1)
    got = M.name_dist32(q, table, name).astype(np.float64)
    want = M.scipy_dist(q, table, name)
    if name in ("cosine", "correlation"):
        np.testing.assert_allclose(got, want, rtol=0, atol=64 * U)
    else:
        assert np.array_equal(got, want.astype(np.float32).astype(np.float64))


@pytest.mark.parametrize("name", M.SCIPY_NAMES)
def test_replay_ranks_as_the_demo(name):
    """The demo's rank(gen_action, metric, k): sorted(range(n), key=lambda j: metric(item_j, action))[:k], a stable
    sort, against the stable argsort of the replay.  For the exact names the ids are equal; cosine and correlation
    round in fp32, so their orders agree wherever scipy's distances are more than the fp32 error apart."""
    rng = np.random.default_rng(12)
    table, q = M.small_ints(rng, (300, 16), -1, 1), M.small_ints(rng, (4, 16), -1, 1)
    f = _scipy_fn(name)
    got = M.name_dist32(q, table, name)
    for r in range(len(q)):
        demo = sorted(range(len(table)), key=lambda j: f(table[j].astype(np.float64), q[r].astype(np.float64)))[:10]
        mine = np.argsort(got[r], kind="stable")[:10]
        if name not in ("cosine", "correlation"):
            assert list(mine) == demo
            continue
        exact = M.scipy_dist(q[r:r + 1], table, name)[0]
        np.testing.assert_allclose(exact[mine], exact[demo], rtol=0, atol=64 * U)
        gaps = np.abs(exact[:, None] - exact[None, :])
        np.fill_diagonal(gaps, np.inf)
        for i, j in enumerate(demo):
            if gaps[j].min() > 64 * U:
                assert mine[i] == j


@pytest.mark.parametrize("name", M.SCIPY_NAMES)
def test_replay_matches_cdist_on_gaussians(name):
    rng = np.random.default_rng(13)
    table = rng.standard_normal((200, 37)).astype(np.float32)
    q = rng.standard_normal((5, 37)).astype(np.float32)
    got = M.name_dist32(q, table, name).astype(np.float64)
    want = M.scipy_dist(q, table, name)
    np.testing.assert_allclose(got, want, rtol=64 * 37 * U, atol=64 * 37 * U)


def test_minkowski_orders_are_the_named_metrics():
    rng = np.random.default_rng(14)
    table, q = M.small_ints(rng, (50, 8)), M.small_ints(rng, (3, 8))
    for p, name in ((1, "cityblock"), (2, "euclidean"), (float("inf"), "chebyshev")):
        np.testing.assert_array_equal(M.name_dist32(q, table, "minkowski", p), M.name_dist32(q, table, name))
        np.testing.assert_allclose(M.scipy_dist(q, table, "minkowski", p), M.scipy_dist(q, table, name))


def test_conventions_where_scipy_gives_nan():
    z = np.zeros((1, 5), np.float32)
    x = np.array([[1, -2, 0, 3, 0.5]], np.float32)
    c = np.full((1, 5), 2.5, np.float32)
    # Bray-Curtis: two zero rows 0 (scipy NaN); t = -q != 0: +inf (scipy's value), ranked and reported as FLT_MAX
    assert M.dist32(z, z, "BRAYCURTIS")[0, 0] == 0
    assert torch.isinf(M.dist64(x, -x, "BRAYCURTIS")[0, 0]) and M.dist32(x, -x, "BRAYCURTIS")[0, 0] == float("inf")
    assert M.name_dist32(x, -x, "braycurtis")[0, 0] == M.FLT_MAX
    with np.errstate(invalid="ignore", divide="ignore"):
        assert np.isinf(M.scipy_dist(x, -x, "braycurtis")[0, 0])
    # Canberra: a zero denominator is a zero term, as scipy has it
    assert M.dist32(z, z, "CANBERRA")[0, 0] == 0 and M.scipy_dist(z, z, "canberra")[0, 0] == 0
    assert M.dist32(x, z, "CANBERRA")[0, 0] == 4.0 == M.scipy_dist(x, z, "canberra")[0, 0]
    # correlation: a constant row (zero included) is at distance 1 from anything (scipy NaN)
    for a, b in ((c, x), (x, c), (z, x), (c, c), (z, z)):
        assert M.dist32(a, b, "CORR")[0, 0] == 1 and M.dist64(a, b, "CORR")[0, 0] == 1
    # a constant row whose fp32 mean is not its value is still constant
    third = np.full((1, 3), 0.1, np.float32)
    mean, norm = M.corr_stats32(third)
    assert mean[0] == third[0, 0] and norm[0] == 0
    # NaN rows: every metric's distance is NaN, so the key is FLT_MAX
    nan = np.array([[1, np.nan, 0, 0, 0]], np.float32)
    for code in M.CODES:
        assert torch.isnan(M.dist32(x, nan, code)[0, 0]) and torch.isnan(M.dist64(x, nan, code)[0, 0]), code
        assert M.finite_key(M.dist32(x, nan, code))[0, 0] == M.FLT_MAX


def test_linf_propagates_nan_and_clipped_corr_keeps_it():
    a = torch.tensor([[0.0, 5.0, 1.0]])
    b = torch.tensor([[float("nan"), 0.0, 0.0]])
    assert torch.isnan(M.dist32(a, b, "LINF")[0, 0])          # fmaxf would drop the NaN and return 5
    assert torch.isnan(M.dist32(a, b, "CORR")[0, 0])


def test_python_refusals():
    t = torch.zeros(4, 3)
    with pytest.raises(ValueError, match="metric must be one of"):
        ItemIndex(t, "hamming")
    with pytest.raises(ValueError, match="metric must be one of"):
        ItemIndex(t, "l1")
    for p in (3, 0.5, -1, float("nan")):
        with pytest.raises(ValueError, match="minkowski"):
            ItemIndex(t, "minkowski", p=p)
    with pytest.raises(ValueError, match="p is minkowski"):
        ItemIndex(t, "cityblock", p=1)
    # the refusals come before the device check: a CPU table with a good name meets the device error instead
    with pytest.raises(_lib.RecnnError):
        ItemIndex(t, "minkowski", p=float("inf"))


@pytest.mark.parametrize("name", ["cityblock", "chebyshev", "canberra", "braycurtis", "correlation", "minkowski"])
def test_ivf_refuses_the_non_l2_metrics(name):
    from recnn_b200.data import db_con
    idx = ItemIndex.__new__(ItemIndex)                       # no device: the refusal needs only the metric
    idx.metric_name = name
    idx.metric = db_con._SCIPY[db_con._metric_name(name, 1 if name == "minkowski" else None)]
    with pytest.raises(ValueError, match="IVF index needs metric"):
        idx.build_ivf(4)
    with pytest.raises(ValueError, match="IVF index needs metric"):
        idx.load_ivf(dict(centroids=None, list_offsets=None, list_ids=None, metric=name, n_items=4, dim=3,
                          params={}))


def test_header_codes_match_the_bindings():
    with open(os.path.join(ROOT, "include", "recnn_b200.h")) as fh:
        h = fh.read()
    codes = dict((k, int(v)) for k, v in re.findall(r"RECNN_METRIC_(\w+)\s*=\s*(\d+)", h))
    assert codes == {"L2": 0, "IP": 1, "COS": 2, "L1": 3, "LINF": 4, "CANBERRA": 5, "BRAYCURTIS": 6, "CORR": 7}
    for k, v in codes.items():
        assert getattr(_lib, "METRIC_" + k) == v
    assert re.search(r"#define RECNN_B200_ABI_VERSION 3\b", h)


def test_c_calls_refuse_before_device_work():
    L = _lib.lib()
    before = L.recnn_b200_launch_count()
    p = 256                                                    # never dereferenced: every call below is refused
    for metric in range(3, 8):
        idx = _lib.IvfIndex(1000, 16, metric, 8, 0, p, p, p, p, p, p)
        a = _lib.IvfSearchArgs(idx, p, 4, 4, 10, None, 0, None, 0, None, p, p, None, p, 1 << 30)
        assert L.recnn_ivf_search(ctypes.byref(a), None) == -1
        b = _lib.IvfBuildArgs(idx, p, p, 500, p, 3, 0, p, 1 << 40)
        assert L.recnn_ivf_build(ctypes.byref(b), None) == -1
        assert L.recnn_ivf_list_table(p, 1000, 16, metric, p, p, p, None) == -1
    # the flat calls: CORR needs its norms, the other new codes do not; 8 and -1 are no metric
    assert L.recnn_retrieve_topk(p, 4, 16, p, 100, None, _lib.METRIC_CORR, 5, p, p, p, 1 << 30, None) == -1
    assert L.recnn_retrieve_rank(p, 4, 16, p, 100, None, _lib.METRIC_CORR, p, p, p, p, 1 << 30, None) == -1
    for metric in (8, -1):
        assert L.recnn_retrieve_topk(p, 4, 16, p, 100, p, metric, 5, p, p, p, 1 << 30, None) == -1
        assert L.recnn_item_norms(p, 100, 16, metric, p, None) == -1
    for metric in (_lib.METRIC_IP, _lib.METRIC_L1, _lib.METRIC_LINF, _lib.METRIC_CANBERRA, _lib.METRIC_BRAYCURTIS):
        assert L.recnn_item_norms(p, 100, 16, metric, p, None) == -1
        # a workspace one byte short is refused after the metric and norms checks pass
        need = L.recnn_retrieve_workspace_bytes(4, 100, 5)
        assert L.recnn_retrieve_topk(p, 4, 16, p, 100, None, metric, 5, p, p, p, need - 1, None) == -3
    assert L.recnn_b200_launch_count() == before


def test_workspace_does_not_depend_on_the_metric():
    L = _lib.lib()
    assert L.recnn_retrieve_workspace_bytes(2048, 1000000, 10) > 0
    assert L.recnn_retrieve_rank_workspace_bytes(2048, 26744) > 0
