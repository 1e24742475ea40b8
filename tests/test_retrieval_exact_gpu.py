"""Item retrieval on exact integer scores: the flat search and rank (recnn_retrieve_topk / _rank and their _sets forms),
the IVF_FLAT fine scan and merge and the IVF_PQ scan, merge and refine must return the stable argsort of the keys, bit
for bit, at the boundaries where a top-k goes wrong: a thread stride, a column range (up to 32 merged by one warp), a
query slab, the 16 -> 64 list switch at k = 17, an IVF list and its work units.

Tables and queries hold integers in [-3, 3], so every score and norm is exact on both GEMM back ends and the oracle of
tests/_exact_retrieval.py reproduces each key and distance in fp32 (scores in float64 on the device).  Integer scores
tie constantly, and copies of a query's best row are planted on both sides of every column-range edge, so a merge that
loses the tie order, or drops or repeats a candidate, changes ids.  Every comparison is equality: ids, ranks, and the
bits of the distances.

NaN and +inf keys rank as FLT_MAX (after every finite key, ties by id) and are returned before any -1 pad, in the
flat search, IVF, IVF_PQ, the critic's top-k and the policy's."""
from __future__ import annotations

import numpy as np
import pytest
import torch

import recnn_b200
from recnn_b200 import _lib
from recnn_b200.data import ItemIndex, ItemSets
from tests import _exact_retrieval as X
from tests.test_ivf_gpu import _device_probes, _lists
from tests.test_workspace_bounds_gpu import check_exact_size, check_too_small

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
L = _lib.lib()
METRICS = ["L2", "IP", "COS"]
KS = [1, 15, 16, 17, 63, 64]
NUM_SMS, TOPK_THREADS = 132, 256           # topk.cuh: kNumSMs, kTopkThreads
FLT_MAX = np.float32(X.FLT_MAX)


def _np(t):
    return t.detach().cpu().numpy()


def _same(a, b):
    """equal arrays; fp32 compared by their bits"""
    a, b = np.asarray(a), np.asarray(b)
    if a.dtype == np.float32 and b.dtype == np.float32:
        a, b = a.view(np.int32), b.view(np.int32)
    return a.shape == b.shape and np.array_equal(a, b)


def _assert_same(got_i, got_d, want_i, want_d, what=""):
    bad = np.nonzero((got_i != want_i).any(1) | (got_d.view(np.int32) != want_d.view(np.int32)).any(1))[0]
    assert bad.size == 0, "%s: %d rows differ, first %d:\n got  %s %s\n want %s %s" % (
        what, bad.size, bad[0], got_i[bad[0]], got_d[bad[0]], want_i[bad[0]], want_d[bad[0]])


# ---------------------------------------------------------------------------------------------- the ranges of a call
def _topk_splits(n_rows, n_items):
    s = min(-(-2 * NUM_SMS // n_rows), -(-n_items // (4 * TOPK_THREADS)), 32)
    return max(s, 1)


def _slab_rows(n_items):
    ld = (n_items + 3) // 4 * 4
    r = (32 << 20) // (ld * 4) // 128 * 128
    return min(max(r, 128), 4096)


def _ranges(n_q, n_items):
    """every (lo, hi) column range of the call's slabs, as retrieval.cu cuts them"""
    slab = min(n_q, _slab_rows(n_items))
    out = set()
    for q0 in range(0, n_q, slab):
        splits = _topk_splits(min(slab, n_q - q0), n_items)
        per = -(-n_items // splits)
        out |= {(sp * per, min(n_items, sp * per + per)) for sp in range(splits) if sp * per < n_items}
    return sorted(out)


def _edge_positions(n_q, n_items):
    """lo - 1, lo and hi - 1 of every range, both sides of the first range's thread stride, and the last range's
    stride when it has one"""
    rs = _ranges(n_q, n_items)
    pos = set()
    for lo, hi in rs:
        pos |= {lo - 1, lo, hi - 1}
    for lo, hi in (rs[0], rs[-1]):
        pos |= {lo + TOPK_THREADS - 1, lo + TOPK_THREADS}
    return sorted(p for p in pos if 0 <= p < n_items)


def _best_row(q, metric):
    """a row that no [-3, 3] row beats for query q: q itself (L2, COS), 3 sign(q) (IP)"""
    return (3.0 * np.sign(q)).astype(np.float32) if metric == "IP" else q.copy()


def _case(n_items, dim, n_q, metric, seed, plant=3):
    """integer table and queries, with copies of the best rows of the first `plant` queries at every range edge"""
    rng = np.random.default_rng(seed)
    table = X.small_ints(rng, (n_items, dim))
    q = X.small_ints(rng, (n_q, dim))
    q[np.abs(q).sum(1) == 0, 0] = 1.0                        # no zero query
    g = min(n_q, plant)
    best = [_best_row(q[i], metric) for i in range(g)]
    for j, p in enumerate(sorted(set(_edge_positions(n_q, n_items)) | {1, n_items - 2})):
        table[p] = best[j % g]
    return table, q


def _dev(x):
    return torch.from_numpy(np.ascontiguousarray(x, dtype=np.float32)).to(DEV)


def _search(index, q, k, **kw):
    res = index.search(q, k, **kw)
    return _np(res.ids), _np(res.distances)


# ------------------------------------------------------------------------------------------------------- flat search
FLAT_CASES = [
    pytest.param(1000, 13, 7, id="cuda-cores-1000x13"),
    pytest.param(1000, 16, 7, id="one-range-1000x16"),
    pytest.param(5000, 64, 1, id="five-ranges-5000x64"),
    pytest.param(33000, 132, 2, id="32-ranges-33000x132"),
    pytest.param(70000, 16, 300, id="three-slabs-70000x16"),
    pytest.param(64, 64, 5, id="k-is-n-64x64"),
]


@pytest.mark.parametrize("metric", METRICS)
@pytest.mark.parametrize("n_items,dim,n_q", FLAT_CASES)
def test_flat_search_and_rank_are_the_stable_argsort(n_items, dim, n_q, metric):
    table, q = _case(n_items, dim, n_q, metric, seed=n_items + dim)
    t, qs = _dev(table), _dev(q)
    index = ItemIndex(t, metric)
    kmax = min(64, n_items)
    want_i, want_d = X.topk(qs, t, metric, kmax)
    assert (np.diff(want_d, axis=1) == 0).any(), "the case has no tie inside the top-k"
    for k in [k for k in KS if k <= kmax]:
        got_i, got_d = _search(index, qs, k)
        _assert_same(got_i, got_d, want_i[:, :k], want_d[:, :k], "k = %d" % k)
    # rank: the position of every returned id, ties included
    for r in range(kmax):
        got = _np(index.rank(qs, torch.from_numpy(want_i[:, r]).to(DEV)))
        assert (got == r).all(), (r, got)
    # random targets, and targets tied with the best row (the planted copies), against the oracle's count
    rng = np.random.default_rng(1)
    edges = _edge_positions(n_q, n_items)
    for target in (rng.integers(0, n_items, n_q), np.asarray(edges)[rng.integers(0, len(edges), n_q)]):
        got = _np(index.rank(qs, torch.from_numpy(target).to(DEV)))
        assert _same(got, X.rank(qs, t, metric, target))


@pytest.mark.parametrize("metric", METRICS)
def test_both_back_ends_return_the_same_bits(metric):
    """dim 64 runs on the tensor cores; the same table or queries at a 4-byte offset force the CUDA-core GEMM"""
    n, dim, n_q = 5000, 64, 9
    table, q = _case(n, dim, n_q, metric, seed=11)
    t, qs = _dev(table), _dev(q)

    def shifted(x):
        buf = torch.empty(x.numel() + 1, device=DEV)[1:].view(x.shape)
        buf.copy_(x)
        return buf
    tc = ItemIndex(t, metric)
    simt = ItemIndex(shifted(t), metric)
    assert simt.table.data_ptr() % 16 == 4 and tc.table.data_ptr() % 16 == 0
    want_i, want_d = X.topk(qs, t, metric, 64)
    target = torch.from_numpy(np.random.default_rng(2).integers(0, n, n_q)).to(DEV)
    want_r = X.rank(qs, t, metric, _np(target))
    for k in (16, 17, 64):
        a = _search(tc, qs, k)
        for b in (_search(simt, qs, k), _search(tc, shifted(qs), k)):
            _assert_same(b[0], b[1], a[0], a[1], "CUDA cores vs tensor cores, k = %d" % k)
        _assert_same(a[0], a[1], want_i[:, :k], want_d[:, :k], "k = %d" % k)
    for idx, qq in ((tc, qs), (simt, qs), (tc, shifted(qs))):
        assert _same(_np(idx.rank(qq, target)), want_r)


# --------------------------------------------------------------------------------------------------------- exclusion
@pytest.mark.parametrize("metric", METRICS)
def test_exclusion_promotes_the_next_ids_of_a_tie_group(metric):
    rng = np.random.default_rng(3)
    n, dim = 2000, 16
    table = X.small_ints(rng, (n, dim))
    q = np.repeat(X.small_ints(rng, (1, dim)), 2, 0)
    q[:, 0] = 2.0
    group = [5, 255, 256, 300, 1024, 1999]                      # both sides of a thread stride, the last item
    table[group] = _best_row(q[0], metric)
    t, qs = _dev(table), _dev(q)
    index = ItemIndex(t, metric)
    sets = [group[:2], []]
    ex = ItemSets.from_lists(sets, device=DEV)
    got_i, got_d = _search(index, qs, 17, exclude=ex)
    assert got_i[0, :4].tolist() == group[2:]
    want_i, want_d = X.topk(qs, t, metric, 17, exclude=sets)
    _assert_same(got_i, got_d, want_i, want_d)
    got_r = _np(index.rank(qs, torch.tensor([1999, 1999], device=DEV), exclude=ex))
    assert got_r.tolist() == [3, 5]

    # fewer than k eligible items: the pads are -1 and FLT_MAX (L2) / -FLT_MAX exactly
    small = X.small_ints(rng, (64, dim))
    small[[3, 9, 40]] = small[9]
    ts = _dev(small)
    keep = [3, 9, 40, 63]
    sets = [[j for j in range(64) if j not in keep], list(range(64))]
    got_i, got_d = _search(ItemIndex(ts, metric), qs, 10, exclude=ItemSets.from_lists(sets, device=DEV))
    want_i, want_d = X.topk(qs, ts, metric, 10, exclude=sets)
    _assert_same(got_i, got_d, want_i, want_d)
    assert sorted(got_i[0, :4].tolist()) == keep and (got_i[0, 4:] == -1).all() and (got_i[1] == -1).all()
    pad = FLT_MAX if metric == "L2" else -FLT_MAX
    assert _same(got_d[0, 4:], np.full(6, pad, np.float32)) and _same(got_d[1], np.full(10, pad, np.float32))


@pytest.mark.parametrize("metric", METRICS)
def test_rank_and_search_with_item_sets_in_shared_and_global_memory(metric):
    """300 queries over 70,000 items (three slabs); set 0 has 3,000 ids (staged in shared memory), set 1 has 5,000
    (searched in global memory), set 2 none"""
    n, dim, n_q = 70000, 16, 300
    table, q = _case(n, dim, n_q, metric, seed=7)
    t, qs = _dev(table), _dev(q)
    index = ItemIndex(t, metric)
    rng = np.random.default_rng(4)
    edges = np.asarray(_edge_positions(n_q, n))
    staged = np.sort(np.concatenate([edges[::2], rng.choice(n, 3000 - len(edges[::2]), replace=False)]))
    staged = np.unique(staged)
    glob = np.unique(np.concatenate([edges[1::2], rng.choice(n, 5000, replace=False)]))
    assert len(staged) <= 4096 < len(glob)
    sets = [staged, glob, np.zeros(0, np.int64)]
    rows = np.arange(n_q) % 3
    per_row = [sets[r] for r in rows]
    ex = ItemSets.from_lists(sets, device=DEV)
    er = torch.from_numpy(rows).to(DEV)
    got_i, got_d = _search(index, qs, 64, exclude=ex, exclude_rows=er)
    want_i, want_d = X.topk(qs, t, metric, 64, exclude=per_row)
    _assert_same(got_i, got_d, want_i, want_d)
    for r in (0, 1, 17, 63):
        got = _np(index.rank(qs, torch.from_numpy(want_i[:, r]).to(DEV), exclude=ex, exclude_rows=er))
        assert (got == r).all(), r
    for target in (rng.integers(0, n, n_q), edges[rng.integers(0, len(edges), n_q)]):
        got = _np(index.rank(qs, torch.from_numpy(target).to(DEV), exclude=ex, exclude_rows=er))
        assert _same(got, X.rank(qs, t, metric, target, exclude=per_row))


# ----------------------------------------------------------------------------------------------------------- IVF_FLAT
def _ivf_case(metric, dim, n=3000, seed=0):
    """integer table; 70 queries: 3 base queries repeated 20 times each (so one list is probed by more than one 32-query
    work unit), then 10 random ones; copies of each base query's best row spread over the table"""
    rng = np.random.default_rng(seed + dim)
    table = X.small_ints(rng, (n, dim))
    base = X.small_ints(rng, (3, dim))
    base[:, 0] = 2.0
    q = np.concatenate([np.repeat(base, 20, 0), X.small_ints(rng, (10, dim))])
    q[np.abs(q).sum(1) == 0, 0] = 1.0
    for b in range(3):
        table[rng.choice(n, 12, replace=False)] = _best_row(base[b], metric)
    return table, q


def _unions(index, qs, nprobe):
    _, offsets, ids = _lists(index)
    probes = _device_probes(index, qs, nprobe)
    return [np.concatenate([ids[offsets[l]:offsets[l + 1]] for l in p if l >= 0]) for p in probes]


@pytest.mark.parametrize("dim", [13, 16])
@pytest.mark.parametrize("metric", METRICS)
def test_ivf_flat_is_the_exact_top_k_of_the_probed_lists(metric, dim):
    table, q = _ivf_case(metric, dim)
    t, qs = _dev(table), _dev(q)
    nlist = 32
    index = ItemIndex(t, metric).build_ivf(nlist, n_iter=5, seed=0)
    flat = ItemIndex(t, metric)
    for k in (17, 64):
        got = _search(index, qs, k, search_param={"nprobe": nlist})
        want = _search(flat, qs, k)
        _assert_same(got[0], got[1], want[0], want[1], "full probe vs flat, k = %d" % k)
        want = X.topk(qs, t, metric, k)
        _assert_same(got[0], got[1], want[0], want[1], "full probe vs oracle, k = %d" % k)
    tied_across_lists = 0
    _, offsets, ids = _lists(index)
    list_of = np.empty(len(table), np.int64)
    list_of[ids] = np.repeat(np.arange(nlist), np.diff(offsets))
    for nprobe in (1, 4, 16):
        unions = _unions(index, qs, nprobe)
        want_i, want_d = X.topk(qs, t, metric, 64, candidates=unions)
        for k in (1, 16, 17, 64):
            got_i, got_d = _search(index, qs, k, search_param={"nprobe": nprobe})
            _assert_same(got_i, got_d, want_i[:, :k], want_d[:, :k], "nprobe %d, k = %d" % (nprobe, k))
        for r in range(len(q)):
            eq = (want_i[r, 1:] >= 0) & (want_d[r, 1:] == want_d[r, :-1])
            tied_across_lists += int((eq & (list_of[want_i[r, 1:]] != list_of[np.maximum(want_i[r, :-1], 0)])).sum())
        # the repeated queries share their lists and their results
        for b in range(3):
            assert (want_i[20 * b:20 * b + 20] == want_i[20 * b]).all()
    assert tied_across_lists > 0, "no tie between two lists inside a top-k"


# ------------------------------------------------------------------------------------------------------------- IVF_PQ
@pytest.mark.parametrize("metric", METRICS)
def test_ivf_pq_duplicate_codes_tie_by_id_and_full_refine_is_exact(metric):
    n, dim, m, nlist = 512, 16, 4, 32
    rng = np.random.default_rng(5)
    table = X.small_ints(rng, (n, dim))
    dups = [7, 100, 255, 256, 400, 511]
    table[dups] = table[7]
    q = np.concatenate([table[7:8], X.small_ints(rng, (23, dim))])
    q[np.abs(q).sum(1) == 0, 0] = 1.0
    t, qs = _dev(table), _dev(q)
    pq = ItemIndex(t, metric).build_ivf(nlist, n_iter=5, seed=0, m=m)
    ivf = ItemIndex(t, metric).build_ivf(nlist, n_iter=5, seed=0)
    _, offsets, ids = _lists(pq)
    pos = np.empty(n, np.int64)
    pos[ids] = np.arange(n)
    codes = _np(pq.pq[1])
    assert all(_same(codes[pos[d]], codes[pos[dups[0]]]) for d in dups), "duplicate rows encode differently"
    lst = np.searchsorted(offsets, pos[dups], side="right") - 1
    assert (lst == lst[0]).all()
    # every item of that list with the same codes has the same ADC key: the duplicates and any item that happens to
    # share their codes.  Wherever the group enters the top-k it is its smallest ids, ascending and adjacent.
    members = ids[offsets[lst[0]]:offsets[lst[0] + 1]]
    group = sorted(int(j) for j in members if _same(codes[pos[j]], codes[pos[dups[0]]]))
    seen = 0
    for nprobe in (1, 4):
        got_i, _ = _search(pq, qs, 20, search_param={"nprobe": nprobe})
        for r in range(len(q)):
            at = np.nonzero(np.isin(got_i[r], group))[0]
            if at.size:
                seen += 1
                assert got_i[r, at].tolist() == group[:at.size], (r, got_i[r])
                assert (np.diff(at) == 1).all(), (r, got_i[r])
    assert seen > 0
    # refine over every eligible item of the probed lists: IVF_FLAT's result and the exact oracle, bit for bit
    covered = 0
    for nprobe, k, refine in ((1, 64, 1), (2, 8, 8)):
        unions = _unions(pq, qs, nprobe)
        rows = np.array([r for r in range(len(q)) if len(unions[r]) <= refine * k])
        covered += len(rows)
        got_i, got_d = _search(pq, qs, k, search_param={"nprobe": nprobe, "refine": refine})
        flat_i, flat_d = _search(ivf, qs, k, search_param={"nprobe": nprobe})
        want_i, want_d = X.topk(qs, t, metric, k, candidates=unions)
        if len(rows):
            _assert_same(got_i[rows], got_d[rows], flat_i[rows], flat_d[rows], "refine vs IVF_FLAT")
            _assert_same(got_i[rows], got_d[rows], want_i[rows], want_d[rows], "refine vs oracle")
        # without refine the ADC top-k of a short union is the whole union
        adc_i, _ = _search(pq, qs, 64, search_param={"nprobe": nprobe})
        for r in range(len(q)):
            if len(unions[r]) <= 64:
                assert sorted(adc_i[r][adc_i[r] >= 0].tolist()) == sorted(unions[r].tolist()), r
    assert covered >= len(q)


# -------------------------------------------------------------------------------------------------------------- scale
def test_million_items_against_the_float64_device_oracle():
    """1,048,576 x 64, k = 64: 1 and 7 queries (32 ranges), 300 (three slabs of 3, 3 and 6 ranges)"""
    n, dim = 1 << 20, 64
    g = torch.Generator(device=DEV).manual_seed(0)
    t = torch.randint(-3, 4, (n, dim), device=DEV, generator=g).to(torch.float32)
    q = torch.randint(-3, 4, (300, dim), device=DEV, generator=g).to(torch.float32)
    q[:, 0] = 3.0
    edges = _edge_positions(1, n) + _edge_positions(7, n) + _edge_positions(300, n)
    t[torch.tensor(edges, device=DEV)] = q[0]
    index = ItemIndex(t, "L2")
    assert [_topk_splits(nq, n) for nq in (1, 7, 128, 44)] == [32, 32, 3, 6] and _slab_rows(n) == 128
    for nq in (1, 7, 300):
        got_i, got_d = _search(index, q[:nq], 64)
        want_i, want_d = X.topk(q[:nq], t, "L2", 64)
        _assert_same(got_i, got_d, want_i, want_d, "%d queries" % nq)
    for r in (0, 31, 32, 63):
        assert (_np(index.rank(q, torch.from_numpy(got_i[:, r]).to(DEV))) == r).all()


# ---------------------------------------------------------------------------------------------------- non-finite keys
def _nonfinite_l2_table(rng, n, dim):
    """integer rows, one holding 2^64 (|t|^2 overflows: key +inf) and two NaN rows"""
    table = X.small_ints(rng, (n, dim))
    table[10, 3] = 2.0 ** 64
    table[[20, n - 1]] = np.nan
    return table, [10, 20, n - 1]


def _overflow_queries(rng, n_q, dim):
    """IP queries 2^126 in dims 0 and 1, 0 elsewhere: <q, t> = 2^126 (t0 + t1), +-inf for |t0 + t1| >= 4"""
    q = np.zeros((n_q, dim), np.float32)
    q[:, :2] = 2.0 ** 126
    q[1::2, 1] = -(2.0 ** 126)
    return q


@pytest.mark.parametrize("dim", [13, 16])
def test_nonfinite_keys_flat_search_and_rank(dim):
    rng = np.random.default_rng(6)
    cases = []
    table, special = _nonfinite_l2_table(rng, 64, dim)
    q = X.small_ints(rng, (5, dim))
    q[:, 3] = 0.0
    cases.append(("L2", table, q))
    table = X.small_ints(rng, (64, dim))
    cases.append(("IP", table, _overflow_queries(rng, 4, dim)))
    for metric, table, q in cases:
        t, qs = _dev(table), _dev(q)
        index = ItemIndex(t, metric)
        want_i, want_d = X.topk(qs, t, metric, 64, bound=None)
        assert (want_i >= 0).all() and (np.abs(want_d) == FLT_MAX).any()
        got_i, got_d = _search(index, qs, 64)
        assert (got_i >= 0).all(), "%s: -1 returned for an eligible item:\n%s" % (metric, got_i)
        _assert_same(got_i, got_d, want_i, want_d, metric)
        for r in (0, 40, 62, 63):
            assert (_np(index.rank(qs, torch.from_numpy(want_i[:, r]).to(DEV))) == r).all(), (metric, r)
    # L2 with exclusion: the two eligible items come back, the FLT_MAX one second, then pads
    t = _dev(cases[0][1])
    keep = [special[0], 33]
    sets = [[j for j in range(64) if j not in keep]] * 5
    got_i, got_d = _search(ItemIndex(t, "L2"), _dev(cases[0][2]), 4, exclude=ItemSets.from_lists(sets, device=DEV))
    assert (got_i == np.array([33, special[0], -1, -1])).all(), got_i
    assert (got_d[:, 1:] == FLT_MAX).all()


def test_nonfinite_keys_ivf_and_ivf_pq():
    """IVF_FLAT probing every list of a 60-item index returns all 60 items at k = 60, the FLT_MAX keys (NaN rows,
    scores that overflow to -inf) after the finite ones.  On 512 items with the overflowing row, NaN rows and
    overflowing queries, IVF_FLAT, IVF_PQ's full refine and its ADC scan return the probed lists' exact top-k."""
    rng = np.random.default_rng(8)
    flt_max_returned = 0
    small_l2 = X.small_ints(rng, (60, 16))
    small_l2[[20, 59]] = np.nan
    for metric, table, q in (("L2", small_l2, X.small_ints(rng, (6, 16))),
                             ("IP", X.small_ints(rng, (60, 16)), _overflow_queries(rng, 6, 16))):
        t, qs = _dev(table), _dev(q)
        ivf = ItemIndex(t, metric).build_ivf(4, n_iter=5, seed=0)
        got_i, got_d = _search(ivf, qs, 60, search_param={"nprobe": 4})
        want_i, want_d = X.topk(qs, t, metric, 60, bound=None)
        assert (got_i >= 0).all(), "%s: -1 returned for an eligible item:\n%s" % (metric, got_i)
        _assert_same(got_i, got_d, want_i, want_d, "%s IVF_FLAT, every list" % metric)
        flt_max_returned += int((np.abs(got_d) == FLT_MAX).sum())
    assert flt_max_returned > 0, "no FLT_MAX key among the items"

    n, dim, nlist = 512, 16, 32
    l2_table, _ = _nonfinite_l2_table(rng, n, dim)
    l2_q = X.small_ints(rng, (12, dim))
    ip_table = X.small_ints(rng, (n, dim))
    ip_q = _overflow_queries(rng, 12, dim)
    for metric, table, q in (("L2", l2_table, l2_q), ("IP", ip_table, ip_q)):
        t, qs = _dev(table), _dev(q)
        ivf = ItemIndex(t, metric).build_ivf(nlist, n_iter=5, seed=0)
        pq = ItemIndex(t, metric).build_ivf(nlist, n_iter=5, seed=0, m=4)
        unions = _unions(ivf, qs, 1)
        assert all(_same(a, b) for a, b in zip(unions, _unions(pq, qs, 1)))
        want_i, want_d = X.topk(qs, t, metric, 64, candidates=unions, bound=None)
        got_i, got_d = _search(ivf, qs, 64, search_param={"nprobe": 1})
        _assert_same(got_i, got_d, want_i, want_d, "%s IVF_FLAT" % metric)
        rows = [r for r in range(len(q)) if len(unions[r]) <= 64]
        assert rows
        got_i, got_d = _search(pq, qs, 64, search_param={"nprobe": 1, "refine": 1})
        _assert_same(got_i[rows], got_d[rows], want_i[rows], want_d[rows], "%s IVF_PQ refine" % metric)
        adc_i, _ = _search(pq, qs, 64, search_param={"nprobe": 1})
        for r in rows:
            assert sorted(adc_i[r][adc_i[r] >= 0].tolist()) == sorted(unions[r].tolist()), (metric, r)


def test_nonfinite_critic_scores_return_every_item_by_id():
    """Q = -inf for every item (linear3.bias = -inf): every key is FLT_MAX, so topk is the k smallest ids and a rank
    counts the smaller ids"""
    S, A, H, I, N = 8, 16, 32, 300, 6
    torch.manual_seed(0)
    critic = recnn_b200.nn.Critic(S, A, H)
    with torch.no_grad():
        critic.linear3.bias.fill_(float("-inf"))
    critic = critic.to(DEV).eval()
    state = torch.randn(N, S, device=DEV)
    items = torch.randn(I, A, device=DEV)
    for k in (5, 17, 64):
        values, ids = critic.topk(state, k, items)
        assert (_np(ids) == np.arange(k)).all(), _np(ids)
    target = torch.tensor([0, 1, 150, 298, 299, 17], device=DEV)
    assert torch.equal(critic.rank(state, target, items), target)
    cand = torch.tensor([[250, 3, 40, -1, 7]] * N, device=DEV)
    _, ids = critic.topk(state, 4, items, candidates=cand)
    assert (_np(ids) == np.array([3, 7, 40, 250])).all()


def test_nonfinite_policy_logits_return_every_item_by_id():
    """the policy's top-k already ranks a -inf logit as FLT_MAX: the reference behaviour for the selectors above"""
    S, H, I, N = 12, 32, 500, 4
    torch.manual_seed(0)
    actor = recnn_b200.nn.DiscreteActor(S, I, H)
    with torch.no_grad():
        actor.linear2.bias.fill_(float("-inf"))
    actor = actor.to(DEV)
    _, ids = actor.topk(torch.randn(N, S, device=DEV), 64)
    assert (_np(ids) == np.arange(64)).all(), _np(ids)


# ------------------------------------------------------------------------------------------------- workspace contract
@pytest.mark.parametrize("metric", [_lib.METRIC_L2, _lib.METRIC_COS])
def test_workspace_bounds_three_slab_search_and_rank(metric):
    nq, items, dim, k = 300, 70000, 16, 17
    table, q = _case(items, dim, nq, "L2", seed=9)
    t, qs = _dev(table), _dev(q)
    norms = torch.empty(items, device=DEV)
    _lib.check(L.recnn_item_norms(t.data_ptr(), items, dim, metric, norms.data_ptr(), _lib.stream_ptr()))
    ids, dist = torch.zeros(nq, k, dtype=torch.int64, device=DEV), torch.zeros(nq, k, device=DEV)
    target = torch.randint(0, items, (nq,), device=DEV)
    rank, flag = torch.zeros(nq, dtype=torch.int64, device=DEV), torch.zeros(1, dtype=torch.int32, device=DEV)

    def search(ptr, nbytes):
        return [L.recnn_retrieve_topk(qs.data_ptr(), nq, dim, t.data_ptr(), items, norms.data_ptr(), metric, k,
                                      ids.data_ptr(), dist.data_ptr(), ptr, nbytes, _lib.stream_ptr())]

    def rank_(ptr, nbytes):
        return [L.recnn_retrieve_rank(qs.data_ptr(), nq, dim, t.data_ptr(), items, norms.data_ptr(), metric,
                                      target.data_ptr(), rank.data_ptr(), flag.data_ptr(), ptr, nbytes,
                                      _lib.stream_ptr())]
    for run, size, state in ((search, L.recnn_retrieve_workspace_bytes(nq, items, k), [ids, dist]),
                             (rank_, L.recnn_retrieve_rank_workspace_bytes(nq, items), [rank, flag])):
        check_exact_size(size, 1, run, state)
        check_too_small(size, run)
