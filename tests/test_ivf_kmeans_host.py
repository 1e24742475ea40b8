"""The fp32 k-means round replay (tests/_kmeans_replay.py) against the float64 oracle of tests/_ivf_oracle.py, and the
details that make it the device's round and not just a k-means round: the split cascade's order and the sequential
member sum."""
from __future__ import annotations

import numpy as np
import pytest

from tests import _ivf_oracle as V
from tests import _kmeans_replay as R


def _oracle_round(x64, c64):
    """one round of _ivf_oracle.lloyd (L2), spelled out so that its assignment and split pairs can be read"""
    a = V.assign(x64, c64)
    counts = np.bincount(a, minlength=len(c64)).astype(np.float64)
    c = c64.copy()
    for l in np.nonzero(counts)[0]:
        c[l] = x64[a == l].mean(0)
    pairs = V.split_empty(c, counts)
    return a, c, counts, pairs


def _dup_points(rng, n, dim, distinct):
    """float32 points: `distinct` random rows, each repeated, plus a little noise on half of them so that both exact
    duplicates (equal initial centroids: empty lists) and generic points occur"""
    rows = rng.standard_normal((distinct, dim))
    x = rows[rng.integers(0, distinct, n)]
    x[: n // 2] += 0.05 * rng.standard_normal((n // 2, dim))
    return x.astype(np.float32)


@pytest.mark.parametrize("dim,nlist", [(1, 6), (5, 40), (12, 17)])
def test_round_matches_float64_oracle(dim, nlist):
    rng = np.random.default_rng(dim)
    x = _dup_points(rng, 400, dim, 12)
    x64 = x.astype(np.float64)
    c64 = x64[rng.permutation(len(x))[:nlist]]
    c64[-2:] = c64[:2]                                   # equal initial centroids: the later ones start empty
    splits = 0
    for _ in range(5):
        a, want, want_counts, want_pairs = _oracle_round(x64, c64)
        got, got_counts, got_pairs = R.round_(x, a, c64.astype(np.float32))
        assert got_pairs == want_pairs
        np.testing.assert_array_equal(got_counts, want_counts.astype(np.float32))
        # the float32 mean is the float64 mean rounded once (2^-24 relative); a centroid moved by s splits is then
        # multiplied s times, each product rounded once in float32 where the oracle keeps float64: at most
        # (s + 1) * 2^-24 relative, and s <= the round's number of splits
        bound = (len(want_pairs) + 1) * R.U * np.abs(want) * (1 + 1e-12)
        assert (np.abs(got.astype(np.float64) - want) <= bound).all()
        splits += len(want_pairs)
        c64 = want
    assert splits >= 2, "the case must exercise the split"


def test_split_cascade_rechooses_the_donor_after_each_halving():
    # counts [0, 4, 4, 0, 0, 1]: list 0 takes donor 1 (4 = 4, the smaller id), leaving [2, 2, 4, 0, 0, 1]; list 3 takes
    # donor 2, leaving [2, 2, 2, 2, 0, 1]; list 4 takes donor 0 (four 2s, the smallest id)
    c = np.arange(6 * 3, dtype=np.float32).reshape(6, 3) + 1
    counts = np.array([0, 4, 4, 0, 0, 1], np.float32)
    before = c.copy()
    pairs = R.split(c, counts)
    assert pairs == [(0, 1), (3, 2), (4, 0)]
    np.testing.assert_array_equal(counts, np.array([1, 2, 2, 2, 1, 1], np.float32))
    up, down = np.float32(1 + 2 ** -10), np.float32(1 - 2 ** -10)
    sign_e = np.array([up, down, up], np.float32)          # dims 0, 2 even: * (1 + eps) on the empty list's copy
    sign_d = np.array([down, up, down], np.float32)
    d1 = before[1] * sign_d
    np.testing.assert_array_equal(c[0], (before[1] * sign_e) * sign_d)   # list 0 was donor to list 4 afterwards
    np.testing.assert_array_equal(c[4], (before[1] * sign_e) * sign_e)
    np.testing.assert_array_equal(c[1], d1)
    np.testing.assert_array_equal(c[3], before[2] * sign_e)
    np.testing.assert_array_equal(c[2], before[2] * sign_d)
    np.testing.assert_array_equal(c[5], before[5])
    # an odd count halves in float32: 3 -> 1.5 and 1.5
    counts = np.array([3, 0], np.float32)
    R.split(np.ones((2, 2), np.float32), counts)
    np.testing.assert_array_equal(counts, np.array([1.5, 1.5], np.float32))


@pytest.mark.parametrize("seed", range(6))
def test_split_agrees_with_oracle_split_empty(seed):
    rng = np.random.default_rng(seed)
    k, dim = 40, 7
    counts = rng.integers(0, 4, k).astype(np.float64)
    counts[rng.integers(0, k)] = 0
    counts[rng.integers(0, k)] = 9
    c = rng.standard_normal((k, dim)).astype(np.float32)
    want_c, want_counts = c.astype(np.float64), counts.copy()
    want_pairs = V.split_empty(want_c, want_counts)
    got_c, got_counts = c.copy(), counts.astype(np.float32)
    got_pairs = R.split(got_c, got_counts)
    assert got_pairs == want_pairs and len(got_pairs) >= 2
    np.testing.assert_array_equal(got_counts, want_counts.astype(np.float32))
    # each of a centroid's s <= len(pairs) products rounds once in float32
    bound = len(want_pairs) * R.U * np.abs(want_c) * (1 + 1e-12)
    assert (np.abs(got_c - want_c) <= bound).all()


def test_update_sums_members_sequentially_in_float64():
    # one list's 32 members in dim 0: 2^60, fifteen 1s, -2^60, fifteen 1s.  Summed one after another the first fifteen
    # 1s vanish into 2^60 and the sum is 15; np.sum's pairwise order gives 29; an fp32 sum gives 15 as well but
    # rounds every partial sum at 2^-24, which dim 1 (1 + 2^-20 added 32 times) tells apart from float64
    col0 = np.array([2.0 ** 60] + [1.0] * 15 + [-2.0 ** 60] + [1.0] * 15)
    col1 = np.full(32, 1.0 + 2.0 ** -20)
    x = np.stack([col0, col1], 1).astype(np.float32)
    assign = np.zeros(32, np.int64)
    c, counts = R.update(x, assign, np.zeros((1, 2), np.float32))
    assert counts[0] == 32
    seq = 0.0
    for v in col0:
        seq += v
    assert seq == 15.0 and np.sum(col0) != seq, "the case must tell the two orders apart"
    assert c[0, 0] == np.float32(15.0 / 32)
    assert c[0, 0] != np.float32(np.sum(col0) / 32)
    assert c[0, 1] == np.float32(np.add.accumulate(col1)[-1] / 32)
    f32 = np.float32(0)
    for v in x[:, 1]:
        f32 = np.float32(f32 + v)
    assert c[0, 1] != np.float32(f32 / np.float32(32)), "the case must tell a float32 sum apart"
    # members keep ascending point order whatever the assignment interleaves, and +0.0 starts the sum
    x2 = np.zeros((64, 2), np.float32)
    x2[0::2] = x
    a2 = np.zeros(64, np.int64)
    a2[1::2] = 1
    c2, _ = R.update(x2, a2, np.zeros((2, 2), np.float32))
    assert R.same_bits(c2[0], c[0])
    neg = R.update(np.full((3, 1), -0.0, np.float32), np.zeros(3, np.int64), np.ones((1, 1), np.float32))[0]
    assert R.same_bits(neg, np.zeros((1, 1), np.float32))
    # an empty list keeps its centroid
    c3, counts3 = R.update(x, assign, np.full((2, 2), 7.0, np.float32))
    assert counts3[1] == 0 and (c3[1] == 7.0).all()


def test_decide_resolves_equal_centroids_by_id_and_flags_near_ties():
    c = np.array([[0.0, 1.0], [2.0, 0.0], [0.0, 1.0], [0.0, 1.0 + 2 ** -20]], np.float32)
    x = np.array([[0.0, 1.5], [1.9, 0.0], [1.0, 0.5]], np.float32)
    a, amb = R.decide(x, c[:3], np.full(3, 1e-3))
    # point 0: centroids 0 and 2 are equal bits, so the tie is the device's: the smaller id
    assert a.tolist() == [0, 1, 0] and not amb[:2].any()
    a, amb = R.decide(x, c, np.full(3, 1e-3))
    assert amb[0] and not amb[1]                         # centroid 3 is a distinct near-tie of point 0
    a, amb = R.decide(x, c, np.zeros(3))
    assert not amb[0] and a[0] == 3                      # 1.5 is nearer 1 + 2^-20 than 1


@pytest.mark.parametrize("dim", [1, 13, 132, 512])
def test_key_bar_covers_fp32_keys(dim):
    # the bar of key_bar against keys computed the CUDA-core way (fp32 fma in ascending d, norms fp32): every fp32
    # key difference must sit within the bar of the float64 one
    rng = np.random.default_rng(dim)
    x = rng.standard_normal((64, dim)).astype(np.float32)
    c = rng.standard_normal((9, dim)).astype(np.float32)
    s = np.zeros((64, 9), np.float32)
    n = np.zeros(9, np.float32)
    for d in range(dim):                                 # a * b + s in float64, then float32: an fma up to rare
        # double roundings, which the bar's 2^-20 units absorb
        s = (x[:, d:d + 1].astype(np.float64) * c[None, :, d] + s).astype(np.float32)
        n = (c[:, d].astype(np.float64) ** 2 + n).astype(np.float32)
    key32 = (-2.0 * s.astype(np.float64) + n[None, :]).astype(np.float32).astype(np.float64)
    key64 = R.sq_dists(x, c) - (x.astype(np.float64) ** 2).sum(1)[:, None]
    err = np.abs((key32 - key32[:, :1]) - (key64 - key64[:, :1]))
    assert (err <= R.key_bar(x, c)[:, None]).all()
