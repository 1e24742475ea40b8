"""The device k-means of the IVF and IVF_PQ builds (ivf_lloyd in csrc/ivf.cu), replayed round by round.

The build is deterministic, so build_ivf(nlist, n_iter=t) returns the state after exactly t rounds of one trajectory.
Each test reads the device's state C_t for t = 0..T and checks C_{t+1} against tests/_kmeans_replay.py run from C_t
itself, so an fp32 near-tie early on cannot make the comparison diverge.

- Coarse L2 and IP: the final pass of the build assigns the items by the call a training round makes (the sample is a
  plain copy of table rows; the same centroids, the same |c|^2), so the lists of build(n_iter=t), restricted to the
  sample, are the device's round-(t + 1) assignment A_t.  C_{t+1} must equal split(update(A_t)) bit for bit.
- Coarse COS trains on unit rows, whose assignment the lists do not show.  It is decided here in float64 from C_t,
  and a round is compared (within a derived bar) when no point is ambiguous.
- PQ codebooks: with nlist 1 and a table [X; -X] of small integers the coarse centroid is exactly 0 from round 1 on,
  so the residuals are exactly X and the codebooks of build(n_iter=t), t >= 1, are one Lloyd trajectory over fixed
  points.  Round 1 is integer arithmetic, exact on both GEMM back ends; a later round is compared bit for bit when
  no point is ambiguous.

dim % 4 picks the GEMM back end of the assignment (13, 1, 11: CUDA cores; 16, 132, 512, 4: tensor cores)."""
from __future__ import annotations

import numpy as np
import pytest
import torch

from recnn_b200.data import ItemIndex
from recnn_b200.data.db_con import ivf_pq_sample, ivf_sample
from tests import _kmeans_replay as R
from tests._exact_retrieval import small_ints

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
T = 6


def _dev(x):
    return torch.from_numpy(np.ascontiguousarray(x, dtype=np.float32)).to(DEV)


def _table(kind, n, dim, seed):
    """iid: N(0, 1) rows.  int: 40 distinct rows of integers in [-3, 3], each repeated, so that the initial centroids
    repeat, equal centroids tie to the smaller id and many lists start empty"""
    rng = np.random.default_rng(seed)
    if kind == "iid":
        return rng.standard_normal((n, dim)).astype(np.float32)
    rows = small_ints(rng, (40, dim))
    return rows[rng.integers(0, len(rows), n)]


def _item_lists(ivf, n_items):
    offs, ids = ivf.list_offsets.cpu().numpy(), ivf.list_ids.cpu().numpy()
    out = np.empty(n_items, np.int64)
    out[ids] = np.repeat(np.arange(len(offs) - 1), np.diff(offs))
    return out


def _trajectory(x, metric, nlist, mppc, m=None, rounds=T):
    """for t = 0..rounds: build_ivf(nlist, n_iter=t) -> (centroids float32, each item's list, codebooks or None)"""
    xd = _dev(x)
    out = []
    for t in range(rounds + 1):
        index = ItemIndex(xd, metric).build_ivf(nlist, n_iter=t, seed=0, max_points_per_centroid=mppc, m=m)
        books = None if m is None else index.pq[0].cpu().numpy()
        out.append((index.ivf.centroids.cpu().numpy(), _item_lists(index.ivf, len(x)), books))
    return out


def _first_difference(got, want, pairs):
    bad = np.nonzero((got.view(np.uint32) != want.view(np.uint32)).any(1))[0]
    return "%d lists differ, first %d: got %s want %s; split pairs %s" % (len(bad), bad[0], got[bad[0]][:4],
                                                                          want[bad[0]][:4], pairs[:8])


# ------------------------------------------------------------------------------------------------ coarse, L2 and IP
COARSE = [   # dim, nlist, table, n_items, max_points_per_centroid
    (1, 7, "iid", 600, 256),
    (13, 48, "iid", 3000, 32),      # 3,000 > 48 * 32: a subsample of 1,536 points
    (16, 48, "iid", 2000, 256),
    (132, 300, "iid", 2400, 256),   # dims past the update kernel's 128 threads, lists past the split kernel's 256
    (512, 7, "iid", 800, 256),
    (16, 1, "iid", 300, 256),
    (1, 48, "int", 2000, 256),
    (13, 300, "int", 3000, 256),    # the split cascade: hundreds of empty lists
    (16, 48, "int", 3000, 16),      # a subsample of 768 points
    (132, 7, "int", 700, 256),
    (512, 300, "int", 1500, 256),
]


@pytest.mark.parametrize("metric", ["L2", "IP"])
@pytest.mark.parametrize("dim,nlist,kind,n,mppc", COARSE)
def test_coarse_rounds_replay_bit_for_bit(metric, dim, nlist, kind, n, mppc):
    x = _table(kind, n, dim, seed=1000 * dim + nlist)
    sample, init = (t.numpy() for t in ivf_sample(n, nlist, 0, mppc))
    points = x[sample]
    traj = _trajectory(x, metric, nlist, mppc)
    assert R.same_bits(traj[0][0], points[init])               # round 0: the initial centroids, gathered
    empties = []
    for t in range(T):
        c_t, lists_t, _ = traj[t]
        a_t = lists_t[sample]
        # A_t is an L2 assignment to C_t: every point is in a list within the near-tie bar of its nearest centroid
        gap, bar = R.gaps(points, c_t, a_t), R.key_bar(points, c_t)
        assert (gap <= bar).all(), "round %d: a point is %g farther than its nearest centroid" % (t + 1, gap.max())
        want, _, pairs = R.round_(points, a_t, c_t)
        got = traj[t + 1][0]
        assert R.same_bits(got, want), "round %d: %s" % (t + 1, _first_difference(got, want, pairs))
        empties.append(len(pairs))
    print("empty lists per round: %s" % empties)
    if (dim, nlist, kind) == (13, 300, "int"):
        assert max(empties) >= 2 and sum(empties) >= 100, empties


# ------------------------------------------------------------------------------------------------ coarse, COS
@pytest.mark.parametrize("dim", [13, 16])
def test_cos_rounds_within_derived_bar(dim):
    n, nlist, rounds = 500, 8, 8
    rng = np.random.default_rng(dim)
    x = rng.standard_normal((n, dim)).astype(np.float32)
    sample, init = (t.numpy() for t in ivf_sample(n, nlist, 0))
    # equal initial centroids 0 and 1: list 1 starts empty, so round 1 splits and renormalises the copies
    x[sample[init[1]]] = x[sample[init[0]]]
    traj = _trajectory(x, "COS", nlist, 256, rounds=rounds)
    p64 = x[sample].astype(np.float64)
    p64 /= np.linalg.norm(p64, axis=1, keepdims=True)
    points = p64.astype(np.float32)
    # The device's unit rows (ivf_gather_kernel: an fma sum of squares in warp order, sqrt, divide, multiply) are
    # within rho = (dim + 8) * 2^-24 of the exact unit rows, element by element relative to 1 >= |p_d|; so are the
    # float32 roundings used here, so the two differ by at most 2 rho * sqrt(dim) as vectors.  Moving a point by d
    # changes the difference of its squared distances to two centroids of norm <= 1 by at most 2 * d * |c_i - c_j|
    # <= 4 d: the assignment bar adds 8 rho * sqrt(dim) to key_bar.
    rho = (dim + 8) * R.U
    clean = partial = split_rounds = 0
    for t in range(rounds):
        c_t, got = traj[t][0], traj[t + 1][0]
        bar = R.key_bar(points, c_t) + 8 * rho * np.sqrt(dim)
        a, ambiguous = R.decide(points, c_t, bar)
        pre, _, pairs = R.round_(points, a, c_t)
        check = np.ones(nlist, bool)
        if ambiguous.any():
            # an ambiguous point may land in any of its candidate lists.  The other lists keep their members; if no
            # list empties (each candidate list keeps an unambiguous member, and the replay splits nothing) no split
            # runs either, and those lists must match
            affected = R.candidates(points, c_t, bar)[ambiguous].any(0)
            kept = np.bincount(a[~ambiguous], minlength=nlist) > 0
            print("round %d: %d ambiguous points, lists %s" % (t + 1, int(ambiguous.sum()), np.nonzero(affected)[0]))
            if pairs or not kept[affected].all():
                continue
            check = ~affected
            partial += 1
        else:
            clean += 1
            split_rounds += bool(pairs)
        norm = np.linalg.norm(pre.astype(np.float64), axis=1)
        want = pre / norm[:, None]
        # Before the renormalisation both sides hold, per element, the mean of the same members from unit rows 2 rho
        # apart, each rounded to float32 (u = 2^-24 each), then multiplied by the same s split factors, each product
        # rounded (u per side): delta <= 2 rho + 2 u + 2 s u, times (1 + 2^-10)^s <= 1.01 for s <= 10.  Dividing by
        # the norm moves a vector by at most 2 |a - b| / |b| <= 2 sqrt(dim) delta / |pre|, and the device's own
        # renormalisation rounds its norm and product by at most (dim + 9) u.
        s = len(pairs)
        assert s <= 10
        delta = 1.01 * (2 * rho + (2 + 2 * s) * R.U)
        tol = 2 * np.sqrt(dim) * delta / norm + (dim + 9) * R.U
        err = np.abs(got.astype(np.float64) - want).max(1)
        bad = check & (err > tol)
        assert not bad.any(), "round %d: list %d off by %g > %g" % (t + 1, bad.argmax(), err[bad.argmax()],
                                                                   tol[bad.argmax()])
    print("rounds without an ambiguous point: %d of %d (%d of them split), partly compared: %d"
          % (clean, rounds, split_rounds, partial))
    assert clean > rounds // 2 and split_rounds >= 1


# ------------------------------------------------------------------------------------------------ PQ codebooks
DSUB_M = [(1, 8), (4, 4), (11, 2)]


@pytest.mark.parametrize("dsub,m", DSUB_M)
def test_pq_codebook_rounds(dsub, m):
    dim = dsub * m
    rng = np.random.default_rng(dsub)
    half = small_ints(rng, (320, dim))
    x = np.concatenate([half, -half])
    n = len(x)
    # nlist 1 and every item in the sample (n <= 1 * 1024): from round 1 on the centroid is the mean of [X; -X],
    # exactly 0, since every partial sum of the ascending member order is an integer
    traj = _trajectory(x, "L2", 1, 1024, m=m)
    for t in range(1, T + 1):
        assert (traj[t][0] == 0).all()
    pq_init = ivf_pq_sample(n, 0).numpy()
    books = [x[pq_init].reshape(256, m, dsub).transpose(1, 0, 2)] + [traj[t][2] for t in range(1, T + 1)]
    empties, clean = [], 0
    for t in range(T):
        ok = True
        round_empties = 0
        for j in range(m):
            pts = np.ascontiguousarray(x[:, j * dsub:(j + 1) * dsub])
            cur = books[t][j]
            if t == 0:
                # integer points and codewords: every key |c|^2 - 2 <x, c> is an integer below 2^11 in magnitude,
                # exact on both back ends (tests/_exact_retrieval.py), so the float64 argmin (ties: smaller code) is
                # the device's
                a = np.argmin(R.sq_dists(pts, cur), axis=1)
            else:
                a, ambiguous = R.decide(pts, cur, R.key_bar(pts, cur))
                if ambiguous.any():
                    ok = False
                    break
            want, _, pairs = R.round_(pts, a, cur)
            round_empties += len(pairs)
            got = books[t + 1][j]
            assert R.same_bits(got, want), "round %d, subspace %d: %s" % (t + 1, j,
                                                                          _first_difference(got, want, pairs))
        if ok:
            clean += 1
            empties.append(round_empties)
    print("dsub %d: rounds replayed %d of %d; empty codewords per replayed round %s" % (dsub, clean, T, empties))
    if dsub == 1:
        assert empties[0] >= 200 * m                           # at most 7 distinct values for 256 codewords
    if dsub == 11:
        assert clean > T // 2                                  # later rounds replayed, not only the exact first


@pytest.mark.parametrize("dsub,m", DSUB_M)
def test_pq_codes_are_the_stable_argmin_at_n_iter_0(dsub, m):
    dim = dsub * m
    rng = np.random.default_rng(10 + dsub)
    rows = small_ints(rng, (60, dim))
    x = rows[rng.integers(0, len(rows), 700)]
    nlist = 3
    index = ItemIndex(_dev(x), "L2").build_ivf(nlist, n_iter=0, seed=0, m=m)
    sample, init = (t.numpy() for t in ivf_sample(len(x), nlist, 0))
    c0 = x[sample[init]]
    assert R.same_bits(index.ivf.centroids.cpu().numpy(), c0)
    # integer keys: the float64 argmin with ties to the smaller id is the device's list of each item
    lists = np.argmin(R.sq_dists(x, c0), axis=1)
    np.testing.assert_array_equal(_item_lists(index.ivf, len(x)), lists)
    res = x - c0[lists]                                         # exact
    pq_init = ivf_pq_sample(len(sample), 0).numpy()
    want_books = res[sample[pq_init]].reshape(256, m, dsub).transpose(1, 0, 2)
    books, codes = (t.cpu().numpy() for t in index.pq)
    assert R.same_bits(books, want_books)
    by_item = np.empty((len(x), m), np.int64)
    by_item[index.ivf.list_ids.cpu().numpy()] = codes
    ties = 0
    for j in range(m):
        d = R.sq_dists(res[:, j * dsub:(j + 1) * dsub], want_books[j])         # exact integers
        want = np.argmin(d, axis=1)
        np.testing.assert_array_equal(by_item[:, j], want)
        ties += int(((d == d.min(1, keepdims=True)).sum(1) > 1).sum())
    print("items with a tied nearest codeword: %d of %d" % (ties, len(x) * m))
    assert ties > 0
