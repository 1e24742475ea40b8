"""Diversified re-ranking on the device: ``diversify`` (recnn_slate_diversify) certified against the float64
restatement (tests/_diversify_oracle.py) at ragged dims, pool sizes on both sides of the single-CTA / cluster split and
an unaligned table; its exact identities (weight 1, orthogonal rows, repeated ids and duplicates, padding, the rank
limit of the DPP, a clustered pool); bit-identity across repeats, batching, row order, padding columns and column
order; errors; the pools of every serving call end to end; and 16,384 pools of 256 over a million items at the memory
of the outputs."""
from __future__ import annotations

import numpy as np
import pytest
import torch

import recnn_b200
from recnn_b200.data import DeviceFrameFeed, HistoryCSR, ItemIndex
from recnn_b200.utils import diversify
from recnn_b200.utils.metrics import slate_metrics
from tests import _diversify_oracle as O

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
METHODS = ("mmr", "dpp")
WEIGHTS = (0.0, 0.3, 0.7, 1.0)
# The fp32 bar.  A similarity is an fp32 dot over D terms of unit-scale rows divided by fp32 norms: its error is of
# order sqrt(D) 2^-24 (2e-6 at D = 1024), so 2e-5 absolute bounds it, and a relevance term w s is exact to 2^-23
# relative.  The DPP's d^2 loses up to one such error per step through the c-vectors, D2_ERR per step, and log d^2
# turns an absolute error e into e / d^2.
SIM_ATOL, REL, D2_ERR = 2e-5, 1e-6, 1e-5


def _w(weight):
    return float(np.float32(weight))          # the weight the kernel sees


def _bars(g, obj):
    """Per-column fp32 bar on the objective, and the bar on d^2, at the current step of g."""
    if g.dpp:
        d2err = D2_ERR * (g.t + 1)
        a2 = g.w / (1 - g.w)
        with np.errstate(divide="ignore"):
            logbar = np.where(g.d2 > 2 * d2err, d2err / np.maximum(g.d2, 1e-300), np.inf)
        return REL * np.abs(a2 * g.s) + SIM_ATOL + logbar, d2err
    return REL * np.abs(g.s) + SIM_ATOL, 0.0


def certify(ids, scores, table, k, method, weight, got_ids, got_pos, got_gain):
    """Replay the kernel's picks of every row in float64: each pick is eligible and within the bar of the best
    objective at its step, its gain within the bar of its float64 objective, and a row ends (-1 / -1 / NaN) only when
    nothing is eligible or (DPP) a near-best column has d^2 below the stopping threshold.  Where every step's gap to the
    best other id exceeds the bar, the row must equal the float64 greedy exactly.  Returns the number of such rows."""
    clear_rows = 0
    for r in range(ids.shape[0]):
        g = O.Greedy(ids[r], scores[r], table, method, _w(weight))
        clear = True
        for t in range(k):
            obj = g.objective()
            bar, d2bar = _bars(g, obj)
            j = int(got_pos[r, t])
            if j < 0:
                assert (got_pos[r, t:] == -1).all() and (got_ids[r, t:] == -1).all(), r
                assert np.isnan(got_gain[r, t:]).all(), r
                b = g.best(obj)
                if b is not None:
                    assert g.dpp, (r, t, "MMR stopped with an eligible column")
                    near = g.alive & (obj >= obj[b] - bar)
                    assert (g.d2[near] < O.DPP_EPS + d2bar).any(), (r, t, g.d2[b])
                    clear &= g.d2[b] < O.DPP_EPS - d2bar
                break
            assert g.alive[j] and got_ids[r, t] == ids[r, j], (r, t, j)
            best = np.nanmax(obj)
            assert obj[j] >= best - bar[j], (r, t, j, obj[j], best, bar[j])
            assert abs(float(got_gain[r, t]) - obj[j]) <= bar[j], (r, t, got_gain[r, t], obj[j], bar[j])
            if g.dpp:
                assert g.d2[j] >= O.DPP_EPS - d2bar, (r, t, g.d2[j])
                clear &= g.d2[j] >= O.DPP_EPS + d2bar
            others = g.alive & (ids[r] != ids[r, j])
            if others.any():
                clear &= obj[j] - np.nanmax(np.where(others, obj, np.nan)) > bar[j] + np.nanmax(np.where(others, bar, 0))
            g.pick(j)
        if clear:
            want = O.greedy(ids[r], scores[r], table, k, method, _w(weight))
            assert np.array_equal(got_ids[r], want[0]) and np.array_equal(got_pos[r], want[1]), r
            clear_rows += 1
    return clear_rows


def _pools(n, m, n_items, seed, empty=0.1):
    rng = np.random.default_rng(seed)
    ids = rng.integers(0, n_items, (n, m))
    ids[rng.random((n, m)) < empty] = -1
    if m >= 4 and n >= 2:
        ids[1, m - 1] = ids[1, 0] = 5                   # a repeated id
        ids[0, :] = -1                                  # an empty pool
    scores = rng.normal(0, 1, (n, m)).astype(np.float32)
    return ids, scores


def _run(ids, scores, table, k, method, weight):
    out = diversify(torch.from_numpy(ids).to(DEV), torch.from_numpy(scores).to(DEV), table, k, method, weight)
    return tuple(t.cpu().numpy() for t in out)


# ----------------------------------------------------------------------------- 1. against float64
# (dim, m, k).  Shared memory per CTA decides the plan: at dim 1024, m = 17 fits one CTA and m = 64 / 256 split over a
# cluster of 4 / 8; at dim 256 / 257, m <= 65 fits one CTA and m = 256 takes a cluster; small pools pack rows per CTA.
SHAPES = [(1, 17, 10), (1, 256, 64), (7, 64, 10), (7, 256, 64), (128, 1, 1), (128, 65, 64), (256, 64, 64),
          (256, 256, 10), (257, 17, 10), (257, 65, 64), (257, 256, 10), (1024, 17, 10), (1024, 64, 64),
          (1024, 256, 10)]


@pytest.mark.parametrize("method", METHODS)
@pytest.mark.parametrize("D,m,k", SHAPES)
def test_against_float64(D, m, k, method):
    n_items = 3000
    table = torch.randn(n_items, D, generator=torch.Generator().manual_seed(D + m)).to(DEV)
    t64 = table.double().cpu().numpy()
    ids, scores = _pools(6, m, n_items, seed=D * 7 + m + k)
    clear = 0
    for weight in WEIGHTS:
        got = _run(ids, scores, table, k, method, weight)
        clear += certify(ids, scores, t64, k, method, weight, *got)
    assert clear >= 4, clear                             # the exact comparison ran on some rows


def test_unaligned_table_takes_the_scalar_path():
    base = torch.randn(1001 * 64 + 1, generator=torch.Generator().manual_seed(3)).to(DEV)
    table = base[1:].view(1001, 64)                      # 4-byte aligned only: no 16-byte copies
    assert table.data_ptr() % 16 != 0
    t64 = table.double().cpu().numpy()
    ids, scores = _pools(9, 40, 1001, 4)
    for method in METHODS:
        got = _run(ids, scores, table, 12, method, 0.5)
        certify(ids, scores, t64, 12, method, 0.5, *got)
        aligned = _run(ids, scores, table.clone(), 12, method, 0.5)
        for a, b in zip(got, aligned):
            assert np.array_equal(a.view(np.int32) if a.dtype == np.float32 else a,
                                  b.view(np.int32) if b.dtype == np.float32 else b)


# ----------------------------------------------------------------------------- 2. exact identities
def _feed(seed=4, F=4, n_users=60, items=400, dim=16):
    rng = np.random.default_rng(seed)
    lengths = rng.integers(F + 1, 40, n_users)
    hist = [rng.integers(0, 150, n) for n in lengths]
    rat = [rng.integers(1, 6, n).astype(np.float32) for n in lengths]
    csr = HistoryCSR(np.arange(n_users), hist, rat, F)
    return DeviceFrameFeed(csr, torch.from_numpy(rng.normal(0, 1, (items, dim)).astype(np.float32)), DEV), hist


def test_weight_one_returns_the_pool_head():
    feed, _ = _feed()
    F, dim, n_items = feed.frame_size, feed.table.shape[1], feed.table.shape[0]
    torch.manual_seed(2)
    policy = recnn_b200.nn.DiscreteActor(F * dim + F, n_items, 32).to(DEV)
    pos = np.arange(feed.csr.n_users)
    v, ids = policy.topk(feed.user_states(pos), 64, exclude=feed.seen_items(),
                         exclude_rows=torch.from_numpy(pos).to(DEV))
    lv = v.log()
    # log pi can round two neighbouring probabilities to one value; such rows follow the tie rule (the smaller id)
    strict = (lv[:, :-1] > lv[:, 1:]).all(1)
    assert bool(strict.any())
    lv_h, ids_h = lv.cpu().numpy(), ids.cpu().numpy()
    order = np.stack([np.lexsort((ids_h[r], -lv_h[r].astype(np.float64))) for r in range(lv.shape[0])])
    for method in METHODS:
        for k in (1, 10, 64):
            got, p, gain = diversify(ids, lv, feed.table, k, method, 1.0)
            assert torch.equal(got[strict], ids[strict, :k]), (method, k)
            assert torch.equal(p[strict], torch.arange(k, device=DEV).expand(int(strict.sum()), k))
            assert np.array_equal(p.cpu().numpy(), order[:, :k]), (method, k)
            assert torch.equal(gain, lv.gather(1, p))


def test_dpp_on_orthogonal_rows_orders_by_score():
    n_items = 300
    table = torch.eye(n_items, device=DEV)
    rng = np.random.default_rng(1)
    ids = np.stack([rng.permutation(n_items)[:40] for _ in range(8)])
    scores = rng.normal(0, 1, ids.shape).astype(np.float32)
    want = np.take_along_axis(ids, np.argsort(-scores, axis=1, kind="stable"), 1)[:, :20]
    for weight in (0.3, 0.7):
        got, _, _ = _run(ids, scores, table, 20, "dpp", weight)
        assert np.array_equal(got, want), weight


def test_repeated_ids_and_duplicate_rows():
    table = torch.randn(50, 32, generator=torch.Generator().manual_seed(0)).to(DEV)
    table[11] = table[10]                                # two ids, one vector
    ids = np.array([[5, 10, 5, 11, 7, 5, 12, 13, 14, 10]] * 2)
    scores = np.array([[3.0, 2.9, 2.8, 2.95, 0.1, 2.7, 0.2, 0.3, 0.4, 1.0],
                       [0.0, 1.0, 2.0, 3.0, 4.0, 5.0, 6.0, 7.0, 8.0, 9.0]], dtype=np.float32)
    for method in METHODS:
        for weight in WEIGHTS:
            got, pos, gain = _run(ids, scores, table, 8, method, weight)
            for r in range(2):
                f = got[r][got[r] >= 0]
                assert len(set(f.tolist())) == f.size, (method, weight, got[r])
                assert np.array_equal(ids[r][pos[r][pos[r] >= 0]], f)
                assert f.size <= 7                       # 7 distinct ids
                if method == "dpp" and weight < 1:
                    assert not (10 in f and 11 in f), got[r]


def test_short_rows_and_dpp_stops_are_padded():
    table = torch.randn(100, 1, generator=torch.Generator().manual_seed(1)).to(DEV)
    table[:50] = table[:50].abs() + 0.1                  # ids < 50 positive, >= 50 negative
    table[50:] = -table[50:].abs() - 0.1
    ids = np.array([[1, 2, 3, 60, 70, 80, -1, -1], [1, 1, -1, -1, -1, -1, -1, 2], [1, 2, 3, 4, 5, 6, 7, 8]])
    scores = np.linspace(1, 0, 24, dtype=np.float32).reshape(3, 8)
    for weight in (0.0, 0.5):
        got, pos, gain = _run(ids, scores, table, 5, "dpp", weight)
        assert (got[0] >= 0).sum() == 2 and {int(got[0, 0]) < 50, int(got[0, 1]) < 50} == {True, False}
        assert (got[2] >= 0).sum() == 1                  # one direction only: rank S = 1 ... after one pick d^2 = 0
        for r in range(3):
            f = int((got[r] >= 0).sum())
            assert (got[r, f:] == -1).all() and (pos[r, f:] == -1).all() and np.isnan(gain[r, f:]).all()
            assert np.isfinite(gain[r, :f]).all()
    got, pos, gain = _run(ids, scores, table, 5, "mmr", 0.5)
    assert got[1].tolist() == [1, 2, -1, -1, -1] and pos[1, 2:].tolist() == [-1] * 3 and np.isnan(gain[1, 2:]).all()
    assert (got[0] >= 0).sum() == 5


def _clustered(n=16, D=16, seed=0):
    """Pools of 10 near-copies of one direction, scored 1.0-1.2, and 10 of an orthogonal one, scored 0.5-0.7."""
    g = torch.Generator().manual_seed(seed)
    table = torch.zeros(40, D)
    table[:20, 0] = 1.0
    table[20:, 1] = 1.0
    table += 0.05 * torch.randn(40, D, generator=g)
    rng = np.random.default_rng(seed)
    ids = np.stack([np.concatenate([rng.choice(20, 10, replace=False), 20 + rng.choice(20, 10, replace=False)])
                    for _ in range(n)])
    scores = np.concatenate([rng.uniform(1.0, 1.2, (n, 10)), rng.uniform(0.5, 0.7, (n, 10))], 1).astype(np.float32)
    return table.to(DEV), ids, scores


def test_clustered_pool():
    table, ids, scores = _clustered()
    for method in METHODS:
        got, _, _ = _run(ids, scores, table, 4, method, 1.0)
        assert (got < 20).all()                          # relevance only: the first cluster
        div, _, _ = _run(ids, scores, table, 4, method, 0.5)
        assert (div[:, 0] < 20).all() and (div[:, 1] >= 20).all(), (method, div)
        ild = lambda s: slate_metrics(torch.from_numpy(s).to(DEV), table)["ild_min"]
        assert ild(div) >= ild(got), method


# ----------------------------------------------------------------------------- 3. bit-identity
def _bits(x):
    return x.view(np.int32) if x.dtype == np.float32 else x


@pytest.mark.parametrize("method", METHODS)
def test_bit_identical_across_repeats_batching_order_padding_and_columns(method):
    n_items, D, m, k = 5000, 256, 60, 24
    table = torch.randn(n_items, D, generator=torch.Generator().manual_seed(9)).to(DEV)
    ids, scores = _pools(200, m, n_items, 9)
    first = _run(ids, scores, table, k, method, 0.6)
    again = _run(ids, scores, table, k, method, 0.6)
    for a, b in zip(first, again):
        assert np.array_equal(_bits(a), _bits(b))
    for r in (1, 77, 199):
        alone = _run(ids[r:r + 1], scores[r:r + 1], table, k, method, 0.6)
        for a, b in zip(alone, first):
            assert np.array_equal(_bits(a[0]), _bits(b[r])), r
    perm = np.random.default_rng(1).permutation(200)
    for a, b in zip(_run(ids[perm], scores[perm], table, k, method, 0.6), first):
        assert np.array_equal(_bits(a), _bits(b[perm]))
    # -1 columns appended: m = 60 fits one CTA, m = 256 runs on a cluster; no output bit may change
    pad_ids = np.concatenate([ids, np.full((200, 256 - m), -1)], 1)
    pad_sc = np.concatenate([scores, np.full((200, 256 - m), np.nan, np.float32)], 1)
    for a, b in zip(_run(pad_ids, pad_sc, table, k, method, 0.6), first):
        assert np.array_equal(_bits(a), _bits(b))
    cperm = np.random.default_rng(2).permutation(m)
    got = _run(ids[:, cperm], scores[:, cperm], table, k, method, 0.6)
    assert np.array_equal(got[0], first[0]) and np.array_equal(_bits(got[2]), _bits(first[2]))
    filled = first[1] >= 0
    assert np.array_equal(ids[:, cperm][np.arange(200)[:, None], np.where(filled, got[1], 0)][filled],
                          first[0][filled])


def test_errors_and_empty_batch():
    table = torch.randn(30, 8, device=DEV)
    sc = torch.zeros(1, 3, device=DEV)
    for bad in (30, -2, 1 << 40):
        with pytest.raises(IndexError):
            diversify(torch.tensor([[1, 2, bad]], device=DEV), sc, table, 2)
    for v in (float("nan"), float("inf"), -float("inf")):
        with pytest.raises(ValueError, match="non-finite"):
            diversify(torch.tensor([[1, 2, 3]], device=DEV), torch.tensor([[0.0, v, 1.0]], device=DEV), table, 2)
    diversify(torch.tensor([[1, -1, 29]], device=DEV), torch.tensor([[0.0, float("nan"), 1.0]], device=DEV), table, 2)
    out = diversify(torch.zeros(0, 10, dtype=torch.int64, device=DEV), torch.zeros(0, 10, device=DEV), table, 4)
    assert all(t.shape == (0, 4) for t in out)


# ----------------------------------------------------------------------------- 4. every serving call, end to end
def test_pools_of_every_serving_call():
    feed, hist = _feed()
    F, dim, n_items = feed.frame_size, feed.table.shape[1], feed.table.shape[0]
    S = F * dim + F
    torch.manual_seed(2)
    policy = recnn_b200.nn.DiscreteActor(S, n_items, 32).to(DEV)
    actor = recnn_b200.nn.Actor(S, dim, 32).to(DEV).eval()
    critic = recnn_b200.nn.Critic(S, dim, 32).to(DEV).eval()
    index = ItemIndex(feed.table, "L2")
    pos = np.arange(feed.csr.n_users)
    pos_t = torch.from_numpy(pos).to(DEV)
    s = feed.user_states(pos)
    seen = feed.seen_items()
    v, i = policy.topk(s, 64, exclude=seen, exclude_rows=pos_t)
    sv, si = policy.sample_topk(s, 32, exclude=seen, exclude_rows=pos_t, seed=5)
    res = index.search(actor(s), topk=64, exclude=seen, exclude_rows=pos_t)
    q, qi = critic.topk(s, 40, index.table, exclude=seen, exclude_rows=pos_t)
    pools = {"topk": (i, v.log()), "sample_topk": (si, sv.log()), "search": (res.id(), -res.dist()),
             "critic": (qi, q)}
    t64 = feed.table.double().cpu().numpy()
    for name, (ids, scores) in pools.items():
        for method in METHODS:
            got, p, gain = diversify(ids, scores, feed.table, 10, method, 0.5)
            g, p_h = got.cpu().numpy(), p.cpu().numpy()
            ids_h = ids.cpu().numpy()
            for r in range(g.shape[0]):
                f = g[r][g[r] >= 0]
                assert set(f.tolist()) <= set(ids_h[r].tolist()), name
                assert not set(f.tolist()) & set(hist[r].tolist()), name
                assert np.array_equal(ids_h[r][p_h[r][: f.size]], f)
            certify(ids_h, scores.cpu().numpy(), t64, 10, method, 0.5, g, p_h, gain.cpu().numpy())


# ----------------------------------------------------------------------------- 5. scale
def test_16k_pools_of_256_over_a_million_items_at_output_memory():
    n_items, D, n, m, k = 1 << 20, 256, 16384, 256, 10
    table = torch.randn(n_items, D, generator=torch.Generator(device=DEV).manual_seed(0), device=DEV)
    ids = torch.randint(-1, n_items, (n, m), generator=torch.Generator(device=DEV).manual_seed(1), device=DEV)
    scores = torch.randn(n, m, generator=torch.Generator(device=DEV).manual_seed(2), device=DEV)
    rows = torch.arange(0, n, 1999, device=DEV)
    ids_h, sc_h = ids[rows].cpu().numpy(), scores[rows].cpu().numpy()
    uniq = np.unique(ids_h[ids_h >= 0])
    t64 = table[torch.from_numpy(uniq).to(DEV)].double().cpu().numpy()
    local = np.where(ids_h >= 0, np.searchsorted(uniq, np.maximum(ids_h, 0)), -1)
    for method in METHODS:
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        got, p, gain = diversify(ids, scores, table, k, method, 0.5)
        torch.cuda.synchronize()
        peak = torch.cuda.max_memory_allocated() - base
        outputs = 2 * n * k * 8 + n * k * 4 + 512        # ids, pos, gain and the flag (one 512-byte block)
        assert peak == outputs, (peak, outputs)          # no [N, m, dim] gather, no workspace
        g, p_h, gain_h = got[rows].cpu().numpy(), p[rows].cpu().numpy(), gain[rows].cpu().numpy()
        g_local = np.where(g >= 0, np.searchsorted(uniq, np.maximum(g, 0)), -1)
        certify(local, sc_h, t64, k, method, 0.5, g_local, p_h, gain_h)
        del got, p, gain
