"""Host-side checks of slate evaluation: the entry point in the header, the library and the ctypes table; the refusals of
the C entry point and of slate_distances / slate_metrics before any device work; the float64 restatement against
scipy's cdist; slate_metrics' definitions by hand and against the restatement; and its all-reduce through a gloo world
of 2.  No kernel is launched."""
from __future__ import annotations

import math
import os
import re
import socket

import numpy as np
import pytest
import torch
from scipy.spatial.distance import cdist

from recnn_b200 import _lib
from recnn_b200.utils.metrics import slate_distances, slate_metrics
from tests import _slate_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_new_symbol_in_header_library_and_ctypes_table():
    with open(os.path.join(ROOT, "include", "recnn_b200.h")) as fh:
        declared = set(re.findall(r"RECNN_API\s+[\w\s\*]+?\b(recnn_\w+)\s*\(", fh.read()))
    L = _lib.lib()
    assert "recnn_slate_distances" in declared and "recnn_slate_distances" in _lib.SIGNATURES
    assert getattr(L, "recnn_slate_distances") is not None
    assert declared <= set(_lib.SIGNATURES), sorted(declared - set(_lib.SIGNATURES))
    assert L.recnn_b200_abi_version() == 3


def test_c_refusals_before_device_work():
    L = _lib.lib()
    fake = 256                                  # never dereferenced: every call below is refused by its checks
    k0 = L.recnn_b200_launch_count()
    ok = (fake, 4, 10, fake, 100, 8, 1, fake, fake, fake, None, fake, None)
    for i, bad in [(2, 0), (2, 65), (6, 2), (6, -1), (5, 0), (4, 0), (1, -1), (0, None), (3, None), (7, None),
                   (8, None), (9, None), (11, None)]:
        args = list(ok)
        args[i] = bad
        assert L.recnn_slate_distances(*args) != 0, (i, bad)
    assert L.recnn_b200_launch_count() == k0


def test_module_refusals_happen_before_device_work():
    L = _lib.lib()
    k0 = L.recnn_b200_launch_count()
    ids = torch.tensor([[0, 1, -1], [2, 2, 3]])
    table = torch.zeros(5, 4)
    for bad in (ids[0], ids.int(), ids.float(), ids.numpy(), torch.zeros(3, 0, dtype=torch.int64),
                torch.zeros(3, 65, dtype=torch.int64)):
        with pytest.raises(ValueError):
            slate_distances(bad, table)
        with pytest.raises(ValueError):
            slate_metrics(bad, n_items=5)
    with pytest.raises(ValueError, match="metric"):
        slate_distances(ids, table, metric="l2")
    with pytest.raises(ValueError, match="metric"):
        slate_metrics(ids, table, metric="cityblock")
    for bad_table in (table.double(), table.half(), torch.zeros(5), torch.zeros(0, 4), torch.zeros(5, 0), None):
        with pytest.raises(ValueError, match="table"):
            slate_distances(ids, bad_table)
    with pytest.raises(ValueError, match="table"):
        slate_metrics(ids, table.double())
    with pytest.raises(ValueError, match="n_items"):
        slate_metrics(ids)
    with pytest.raises(ValueError, match="n_items"):
        slate_metrics(ids, n_items=0)
    with pytest.raises(ValueError, match="popularity"):
        slate_metrics(ids, n_items=5, popularity=torch.ones(4, dtype=torch.int64), n_users=3)
    with pytest.raises(ValueError, match="popularity"):
        slate_metrics(ids, n_items=5, popularity=torch.ones(5), n_users=3)
    with pytest.raises(ValueError, match="n_users"):
        slate_metrics(ids, n_items=5, popularity=torch.ones(5, dtype=torch.int64))
    if torch.cuda.is_available():
        with pytest.raises(ValueError, match="device"):
            slate_distances(ids, table.cuda())
    with pytest.raises(_lib.RecnnError, match="CUDA only"):          # no CPU path behind the kernel
        slate_distances(ids, table)
    with pytest.raises(_lib.RecnnError, match="CUDA only"):
        slate_metrics(ids, table)
    with pytest.raises(IndexError):
        slate_metrics(torch.tensor([[0, 5]]), n_items=5)
    with pytest.raises(IndexError):
        slate_metrics(torch.tensor([[0, -2]]), n_items=5)
    assert L.recnn_b200_launch_count() == k0


# ----------------------------------------------------------------------------- the float64 restatement
@pytest.mark.parametrize("metric", ["euclidean", "cosine"])
@pytest.mark.parametrize("D", [1, 7, 64])
def test_restatement_equals_scipy_cdist(metric, D):
    rng = np.random.default_rng(D)
    table = rng.normal(0, 1, (40, D))
    n, k = 30, 12
    ids = rng.integers(0, 40, (n, k))
    ids[rng.random((n, k)) < 0.2] = -1
    ids[3, :] = -1
    ids[4, 1:] = -1
    ids[4, 0] = 3
    ids[5, 5] = ids[5, 2] = 17                                   # a repeated id
    got = O.distance_matrices(ids, table, metric)
    for r in range(n):
        f = np.nonzero(ids[r] >= 0)[0]
        want = cdist(table[ids[r, f]], table[ids[r, f]], metric)
        np.testing.assert_allclose(got[r][np.ix_(f, f)], want, rtol=1e-12, atol=1e-12)
        e = np.nonzero(ids[r] < 0)[0]
        assert np.isnan(got[r][e, :]).all() and np.isnan(got[r][:, e]).all()
    assert got[5, 5, 2] == pytest.approx(0.0, abs=1e-15)              # exactly 0 for euclidean; 1 - 1 +- ulp for cosine
    mean, mn, count = O.row_stats(ids, got)
    assert count[3] == 0 and count[4] == 1 and np.isnan(mean[3:5]).all() and np.isnan(mn[3:5]).all()
    assert mn[5] == pytest.approx(0.0, abs=1e-15)


def test_restatement_zero_vector_has_cosine_distance_one():
    table = np.array([[0.0, 0.0], [1.0, 0.0], [0.0, 2.0]])
    m = O.distance_matrices(np.array([[0, 1, 2, 0]]), table, "cosine")[0]
    assert m[0, 1] == m[1, 0] == m[0, 3] == m[0, 2] == 1.0           # zero with non-zero, and with itself
    assert m[1, 2] == 1.0 and m[0, 0] == 0.0


# ----------------------------------------------------------------------------- slate_metrics by hand
def test_uniform_exposure_and_a_single_item():
    n = 8
    u = slate_metrics(torch.arange(16).reshape(4, 4) % n, n_items=n)
    assert u["gini"] == pytest.approx(0.0, abs=1e-15) and u["exposure_entropy"] == pytest.approx(3.0, rel=1e-15)
    assert u["coverage"] == 1.0 and u["rows"] == 4 and u["slots"] == 16
    one = slate_metrics(torch.full((5, 3), 6, dtype=torch.int64), n_items=n)
    assert one["gini"] == pytest.approx((n - 1) / n, rel=1e-15) and one["exposure_entropy"] == 0.0
    assert one["coverage"] == 1 / n
    half = slate_metrics(torch.tensor([[0, 1, -1], [-1, 0, 1]]), n_items=4)
    assert half["coverage"] == 0.5 and half["slots"] == 4 and half["exposure_entropy"] == 1.0
    assert half["gini"] == pytest.approx(0.5, rel=1e-15)             # (-3 -1 + 1*2 + 3*2) / (4 * 4)
    empty = slate_metrics(torch.full((2, 3), -1, dtype=torch.int64), n_items=4)
    assert empty["coverage"] == 0 and math.isnan(empty["gini"]) and math.isnan(empty["exposure_entropy"])
    assert empty["slots"] == 0 and empty["rows"] == 2


def test_novelty_with_unseen_items():
    pop = torch.tensor([0, 3, 7, 0])
    m = slate_metrics(torch.tensor([[0, 1], [2, -1], [3, 3]]), popularity=pop, n_users=7)
    want = np.mean([-math.log2(1 / 8), -math.log2(4 / 8), -math.log2(8 / 8), -math.log2(1 / 8), -math.log2(1 / 8)])
    assert m["novelty"] == pytest.approx(want, rel=1e-15) and m["slots"] == 5
    assert math.isnan(slate_metrics(torch.full((1, 2), -1, dtype=torch.int64), popularity=pop, n_users=7)["novelty"])


def test_metrics_against_the_restatement():
    rng = np.random.default_rng(3)
    n_items = 200
    ids = rng.zipf(1.5, (64, 10)) - 1
    ids[ids >= n_items] = -1
    pop = rng.integers(0, 50, n_items)
    got = slate_metrics(torch.from_numpy(ids), n_items=n_items, popularity=torch.from_numpy(pop), n_users=60)
    want = O.slate_metrics(ids, n_items, popularity=pop, n_users=60)
    assert set(got) == set(want)
    for key in want:
        assert got[key] == pytest.approx(want[key], rel=1e-12), key


# ----------------------------------------------------------------------------- data-parallel ranks
def _ids(seed=11):
    rng = np.random.default_rng(seed)
    ids = rng.integers(-1, 300, (97, 16))
    return ids, rng.integers(0, 40, 300)


def _gloo_worker(rank, world, port, q):
    import torch.distributed as dist
    dist.init_process_group("gloo", init_method="tcp://127.0.0.1:%d" % port, rank=rank, world_size=world)
    try:
        ids, pop = _ids()
        part = slice(0, 40) if rank == 0 else slice(40, 97)
        q.put((rank, slate_metrics(torch.from_numpy(ids[part]), n_items=300, popularity=torch.from_numpy(pop),
                                   n_users=40, group=dist.group.WORLD)))
    finally:
        dist.destroy_process_group()


def test_group_all_reduce_over_gloo_equals_one_process():
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
    ids, pop = _ids()
    want = slate_metrics(torch.from_numpy(ids), n_items=300, popularity=torch.from_numpy(pop), n_users=40)
    assert want["rows"] == 97
    for k in want:
        assert got[0][k] == pytest.approx(want[k], rel=1e-12) and got[1][k] == got[0][k], k
