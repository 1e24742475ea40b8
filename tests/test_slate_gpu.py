"""Slate evaluation on the device: ``slate_distances`` (recnn_slate_distances) against the float64 restatement
(tests/_slate_oracle.py) at ragged dims and every tile shape, its exact contract (empty slots, repeated ids, zero
vectors, the matrix, errors, bit-identity across repeats and batching), ``slate_metrics`` on the slates of every
serving call, ``DeviceFrameFeed.item_popularity``, and a 16,384-row slate batch over a million items at the memory of
its outputs."""
from __future__ import annotations

import numpy as np
import pytest
import torch

import recnn_b200
from recnn_b200.data import DeviceFrameFeed, HistoryCSR, ItemIndex
from recnn_b200.utils.metrics import slate_distances, slate_metrics
from tests import _slate_oracle as O

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
METRICS = ("euclidean", "cosine")
# The fp32 bar.  Each pair is one fp32 accumulation over D terms of unit-scale rows, whose relative error is of order
# sqrt(D) * 2^-24 (2e-6 at D = 1290); euclidean is compared relative to the distance, cosine (a value in [0, 2])
# absolutely.  Means are fp64 sums of the fp32 pair distances, so they carry the same bar.
EUCLID_RTOL, EUCLID_ATOL, COSINE_ATOL = 2e-5, 1e-6, 2e-5


def _table(n_items, D, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(n_items, D, generator=g).to(DEV)


def _ids(n, k, n_items, seed, empty=0.15):
    rng = np.random.default_rng(seed)
    ids = rng.integers(0, n_items, (n, k))
    ids[rng.random((n, k)) < empty] = -1
    if k >= 3 and n >= 2:
        ids[1, k - 1] = ids[1, 0] = 5                  # a repeated id
    return ids


def _close(got, want, metric):
    got = np.asarray(got, dtype=np.float64)
    nan = np.isnan(want)
    assert np.array_equal(np.isnan(got), nan)
    if metric == "euclidean":
        np.testing.assert_allclose(got[~nan], want[~nan], rtol=EUCLID_RTOL, atol=EUCLID_ATOL)
    else:
        np.testing.assert_allclose(got[~nan], want[~nan], rtol=0, atol=COSINE_ATOL)


def _bits(t):
    return t.contiguous().view(torch.int32)


# ----------------------------------------------------------------------------- 1. against float64
@pytest.mark.parametrize("metric", METRICS)
@pytest.mark.parametrize("D", [1, 7, 128, 256, 257, 1290])
@pytest.mark.parametrize("k", [1, 2, 10, 17, 64])
def test_against_float64(metric, D, k):
    n_items = 300
    table = _table(n_items, D, D * 100 + k)
    t64 = table.double().cpu().numpy()
    for n in (1, 23):
        ids = _ids(n, k, n_items, seed=D + k + n)
        mean, mn, count, mat = slate_distances(torch.from_numpy(ids).to(DEV), table, metric, matrix=True)
        want_m = O.distance_matrices(ids, t64, metric)
        want_mean, want_min, want_count = O.row_stats(ids, want_m)
        _close(mat.cpu(), want_m, metric)
        _close(mean.cpu(), want_mean, metric)
        _close(mn.cpu(), want_min, metric)
        assert np.array_equal(count.cpu().numpy(), want_count)


def test_unaligned_table_rows_take_the_scalar_path():
    base = _table(301 * 64 + 1, 1, 3).reshape(-1)
    table = base[1:].view(301, 64)                  # 4-byte aligned only: the kernel may not use 16-byte copies
    assert table.data_ptr() % 16 != 0
    ids = _ids(9, 12, 301, 4)
    t64 = table.double().cpu().numpy()
    for metric in METRICS:
        mean, mn, count = slate_distances(torch.from_numpy(ids).to(DEV), table, metric)
        want_mean, want_min, _ = O.row_stats(ids, O.distance_matrices(ids, t64, metric))
        _close(mean.cpu(), want_mean, metric)
        _close(mn.cpu(), want_min, metric)


# ----------------------------------------------------------------------------- 2. the contract
@pytest.mark.parametrize("metric", METRICS)
def test_empty_slots(metric):
    table = _table(50, 16, 1)
    ids = torch.tensor([[-1, -1, 3, 4, 9],       # leading
                        [3, 4, 9, -1, -1],       # trailing
                        [-1, -1, -1, -1, -1],    # whole row
                        [-1, 7, -1, -1, -1],     # one filled slot
                        [3, -1, 4, -1, 9]], device=DEV)
    mean, mn, count, mat = slate_distances(ids, table, metric, matrix=True)
    assert count.tolist() == [3, 3, 0, 1, 3]
    assert torch.isnan(mean[2:4]).all() and torch.isnan(mn[2:4]).all()
    assert torch.equal(_bits(mean[0]), _bits(mean[1])) and torch.equal(_bits(mean[0]), _bits(mean[4]))
    assert torch.equal(_bits(mn[0]), _bits(mn[1])) and torch.equal(_bits(mn[0]), _bits(mn[4]))
    assert torch.isnan(mat[2]).all() and torch.isnan(mat[0, :2]).all() and torch.isnan(mat[0, :, :2]).all()
    assert mat[3, 1, 1] == 0 and torch.isnan(mat[3, 0, 0])


@pytest.mark.parametrize("metric", METRICS)
@pytest.mark.parametrize("D", [7, 256])
def test_repeated_id_gives_exactly_zero(metric, D):
    table = _table(100, D, D)
    ids = torch.tensor([[11, 40, 12, 40, 77], [3, 3, -1, -1, -1]], device=DEV)
    mean, mn, count, mat = slate_distances(ids, table, metric, matrix=True)
    assert mn.tolist() == [0.0, 0.0] and mat[0, 1, 3] == 0 and mat[0, 3, 1] == 0 and mean[1] == 0


def test_zero_vector_has_cosine_distance_one():
    table = _table(20, 9, 2)
    table[4] = 0
    ids = torch.tensor([[4, 1, 2], [4, 4, -1]], device=DEV)
    mean, mn, count, mat = slate_distances(ids, table, "cosine", matrix=True)
    assert mat[0, 0, 1] == 1 and mat[0, 0, 2] == 1 and mat[1, 0, 1] == 1 and mean[1] == 1
    assert torch.isfinite(mean).all()


@pytest.mark.parametrize("metric", METRICS)
@pytest.mark.parametrize("k", [5, 17, 64])
def test_matrix_is_symmetric_and_reduces_to_the_row_outputs(metric, k):
    table = _table(500, 100, k)
    ids = _ids(40, k, 500, k)
    mean, mn, count, mat = slate_distances(torch.from_numpy(ids).to(DEV), table, metric, matrix=True)
    assert torch.equal(_bits(mat), _bits(mat.transpose(1, 2)))
    m = mat.cpu().double().numpy()
    filled = ids >= 0
    for r in range(40):
        f = np.nonzero(filled[r])[0]
        assert (np.diagonal(m[r])[f] == 0).all()
        iu = np.triu_indices(k, 1)
        v = m[r][iu]
        v = v[~np.isnan(v)]
        assert v.size == len(f) * (len(f) - 1) // 2
        if v.size:
            assert float(mn[r]) == v.min()
            assert float(mean[r]) == pytest.approx(v.sum() / v.size, rel=1e-6)
    plain = slate_distances(torch.from_numpy(ids).to(DEV), table, metric)
    for a, b in zip(plain, (mean, mn, count)):
        assert torch.equal(_bits(a) if a.dtype == torch.float32 else a, _bits(b) if b.dtype == torch.float32 else b)


def test_out_of_range_id_raises():
    table = _table(30, 8, 0)
    for bad in (30, -2, 1 << 40):
        with pytest.raises(IndexError):
            slate_distances(torch.tensor([[1, 2, bad]], device=DEV), table)
        with pytest.raises(IndexError):
            slate_metrics(torch.tensor([[1, 2, bad]], device=DEV), table)
    slate_distances(torch.tensor([[1, 2, 29]], device=DEV), table)          # the last item is in range


@pytest.mark.parametrize("metric", METRICS)
def test_bit_identical_across_repeats_and_batching(metric):
    table = _table(2000, 257, 9)
    ids = torch.from_numpy(_ids(300, 37, 2000, 9)).to(DEV)
    first = slate_distances(ids, table, metric, matrix=True)
    again = slate_distances(ids, table, metric, matrix=True)
    for a, b in zip(first, again):
        assert torch.equal(a.view(torch.int32), b.view(torch.int32))
    for r in (0, 1, 150, 299):
        alone = slate_distances(ids[r:r + 1].clone(), table, metric, matrix=True)
        for a, b in zip(alone, first):
            assert torch.equal(a[0].view(torch.int32), b[r].view(torch.int32)), r
    perm = torch.randperm(300, generator=torch.Generator().manual_seed(1)).to(DEV)
    shuffled = slate_distances(ids[perm], table, metric)
    for a, b in zip(shuffled, first):
        assert torch.equal(a.view(torch.int32), b[perm].view(torch.int32))


def test_empty_batch():
    mean, mn, count = slate_distances(torch.zeros(0, 10, dtype=torch.int64, device=DEV), _table(5, 4, 0))
    assert mean.shape == mn.shape == count.shape == (0,)


# ----------------------------------------------------------------------------- 3. every serving call, end to end
def _feed(seed=4, F=4, n_users=60, items=400, dim=16):
    rng = np.random.default_rng(seed)
    lengths = rng.integers(F + 1, 40, n_users)
    hist = [rng.integers(0, 150, n) for n in lengths]
    rat = [rng.integers(1, 6, n).astype(np.float32) for n in lengths]
    csr = HistoryCSR(np.arange(n_users), hist, rat, F)
    return DeviceFrameFeed(csr, torch.from_numpy(rng.normal(0, 1, (items, dim)).astype(np.float32)), DEV), hist


def test_item_popularity_against_numpy():
    feed, hist = _feed()
    pop = feed.item_popularity()
    want = np.zeros(feed.table.shape[0], dtype=np.int64)
    for h in hist:
        want[np.unique(h)] += 1
    assert pop.dtype == torch.int64 and pop.device == feed.table.device
    assert np.array_equal(pop.cpu().numpy(), want)
    assert feed.item_popularity() is pop


def test_slates_of_every_serving_call_against_float64():
    feed, hist = _feed()
    F, dim, n_items = feed.frame_size, feed.table.shape[1], feed.table.shape[0]
    S = F * dim + F
    torch.manual_seed(2)
    policy = recnn_b200.nn.DiscreteActor(S, n_items, 32).to(DEV)
    actor = recnn_b200.nn.Actor(S, dim, 32).to(DEV).eval()
    critic = recnn_b200.nn.Critic(S, dim, 32).to(DEV).eval()
    with torch.no_grad():
        critic.linear3.weight.uniform_(-0.3, 0.3)
    index = ItemIndex(feed.table, "L2")
    pos = np.arange(feed.csr.n_users)
    pos_t = torch.from_numpy(pos).to(DEV)
    s = feed.user_states(pos)
    seen = feed.seen_items()
    slates = {
        "topk": policy.topk(s, 10, exclude=seen, exclude_rows=pos_t)[1],
        "sample_topk": policy.sample_topk(s, 10, exclude=seen, exclude_rows=pos_t, seed=5)[1],
        "search": index.search(actor(s), topk=20, exclude=seen, exclude_rows=pos_t).id(),
        "critic": critic.topk(s, 10, index.table, exclude=seen, exclude_rows=pos_t)[1],
    }
    pop, n_users = feed.item_popularity(), feed.csr.n_users
    t64 = feed.table.double().cpu().numpy()
    for name, ids in slates.items():
        assert ids.dtype == torch.int64 and ids.device == feed.table.device
        ids_h = ids.cpu().numpy()
        for metric in METRICS:
            got = slate_metrics(ids, table=feed.table, metric=metric, popularity=pop, n_users=n_users)
            want = O.slate_metrics(ids_h, n_items, t64, metric, pop.cpu().numpy(), n_users)
            assert set(got) == set(want), name
            for key in ("coverage", "gini", "exposure_entropy", "novelty", "rows", "slots"):
                assert got[key] == pytest.approx(want[key], rel=1e-12), (name, key)
            for key in ("ild", "ild_min"):
                assert got[key] == pytest.approx(want[key], rel=EUCLID_RTOL, abs=COSINE_ATOL), (name, metric, key)
    # sampling reaches past the policy's top ranks: its slates cover at least as much of the catalogue
    assert slate_metrics(slates["sample_topk"], n_items=n_items)["coverage"] >= \
        slate_metrics(slates["topk"], n_items=n_items)["coverage"]


# ----------------------------------------------------------------------------- 4. scale
def test_16k_slates_of_64_over_a_million_items_at_output_memory():
    n_items, D, n, k = 1 << 20, 256, 16384, 64
    table = torch.randn(n_items, D, generator=torch.Generator(device=DEV).manual_seed(0), device=DEV)
    ids = torch.randint(-1, n_items, (n, k), generator=torch.Generator(device=DEV).manual_seed(1), device=DEV)
    rows = np.arange(0, n, 997)
    ids_h = ids[torch.from_numpy(rows).to(DEV)].cpu().numpy()
    t64 = table[torch.from_numpy(np.unique(ids_h[ids_h >= 0])).to(DEV)].double().cpu().numpy()
    remap = {v: i for i, v in enumerate(np.unique(ids_h[ids_h >= 0]))}
    local = np.vectorize(lambda v: remap.get(v, -1))(ids_h)
    for metric in METRICS:
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        mean, mn, count = slate_distances(ids, table, metric)
        torch.cuda.synchronize()
        peak = torch.cuda.max_memory_allocated() - base
        outputs = 3 * n * 4 + 512                  # mean, min, count and the error flag (one 512-byte block)
        assert peak <= outputs, (peak, outputs)      # no [N, k, D] gather, no [N, k, k] matrix
        want_mean, want_min, want_count = O.row_stats(local, O.distance_matrices(local, t64, metric))
        _close(mean[torch.from_numpy(rows).to(DEV)].cpu(), want_mean, metric)
        _close(mn[torch.from_numpy(rows).to(DEV)].cpu(), want_min, metric)
        assert np.array_equal(count[torch.from_numpy(rows).to(DEV)].cpu().numpy(), want_count)
        del mean, mn, count
