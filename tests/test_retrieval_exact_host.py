"""The exact-integer retrieval oracle (tests/_exact_retrieval.py) on the CPU: its ranking against scipy and a float64
brute force, its fp32 key replication, and the rule for NaN and +inf keys."""
import numpy as np
import pytest
import torch

from tests import _exact_retrieval as X

FLT_MAX = np.float32(X.FLT_MAX)


def _case(seed, n_items=300, dim=13, n_q=6):
    rng = np.random.default_rng(seed)
    return X.small_ints(rng, (n_items, dim)), X.small_ints(rng, (n_q, dim)), rng


@pytest.mark.parametrize("metric", ["L2", "IP", "COS"])
def test_ranking_matches_scipy_and_float64_brute_force(metric):
    from scipy.spatial import distance
    table, q, _ = _case(1)
    table[0] = 0.0                                  # a zero row: COS norm 1 / 1e-30, key -0 * 1e30
    k = 40
    ids, dist = X.topk(q, table, metric, k)
    rk = X.rank(q, table, metric, np.arange(len(q)) * 7)
    t64 = table.astype(np.float64)
    for i in range(len(q)):
        if metric == "L2":
            v = np.array([distance.sqeuclidean(t, q[i]) for t in t64])
        elif metric == "IP":
            v = -(t64 @ q[i])
        else:
            # the device ranks -<q, t> / |t| (the query's norm only finishes the distance); a zero row scores 0
            v = -(t64 @ q[i]) / np.maximum(np.linalg.norm(t64, axis=1), 1e-30)
        want = np.argsort(v, kind="stable")
        if metric == "COS":
            # scipy's cosine on the rows that are not zero gives the same order as the key (|q| is a common factor)
            nz = want[want != 0]
            sc = np.array([distance.cosine(t64[j], q[i]) for j in nz])
            assert (np.diff(sc) >= -1e-12).all()
        # distinct float64 values are distinct fp32 keys here, and equal ones stay equal: the orders agree exactly,
        # except that COS keys of different rows may round to one fp32 value
        if metric != "COS":
            assert np.array_equal(ids[i], want[:k])
            t = i * 7
            assert rk[i] == int(((v < v[t]) | ((v == v[t]) & (np.arange(len(v)) < t))).sum())
        else:
            vv = v[ids[i]]
            assert (np.diff(vv) >= -1e-6).all()
        if metric == "L2":
            np.testing.assert_array_equal(dist[i], v[want[:k]].astype(np.float32))
        elif metric == "IP":
            np.testing.assert_array_equal(dist[i], (-v[want[:k]]).astype(np.float32))


def test_fp32_key_replication():
    """every key and distance is one IEEE fp32 operation on exact operands, the instruction the device runs"""
    table, q, _ = _case(2, n_items=50, dim=16, n_q=3)
    s = q.astype(np.float64) @ table.astype(np.float64).T
    n = (table.astype(np.float64) ** 2).sum(1)
    s32, n32 = s.astype(np.float32), n.astype(np.float32)
    assert np.array_equal(s32, s) and np.array_equal(n32, n)
    st = X.scores64(q, table)
    np.testing.assert_array_equal(X.keys32(st, X.norms32(table, "L2"), "L2").numpy(), (n32[None] - 2 * s32))
    np.testing.assert_array_equal(X.keys32(st, None, "IP").numpy(), -s32)
    inv = (np.float32(1) / np.sqrt(n32)).astype(np.float32)
    np.testing.assert_array_equal(X.norms32(table, "COS").numpy(), inv)
    np.testing.assert_array_equal(X.keys32(st, X.norms32(table, "COS"), "COS").numpy(), (-s32 * inv[None]))
    key = torch.tensor([[-3.0, 0.25]], dtype=torch.float32)
    qn = torch.tensor([4.0], dtype=torch.float32)
    np.testing.assert_array_equal(X.finish32(key, qn, "L2").numpy(), [[1.0, 4.25]])
    np.testing.assert_array_equal(X.finish32(key, qn, "COS").numpy(), [[1.5, -0.125]])
    np.testing.assert_array_equal(X.finish32(key, qn, "IP").numpy(), [[3.0, -0.25]])
    # the key of an inexact product is rounded once, as the device's fmul / fma round it
    s1 = torch.tensor([[1.0]], dtype=torch.float64)
    cos = X.keys32(s1, torch.tensor([1.0 / 3.0], dtype=torch.float32), "COS")
    assert cos.item() == -np.float32(1.0 / 3.0)


def test_bound_is_asserted():
    table = np.full((2, 4), 30.0, np.float32)               # |t|^2 = 3600 >= 2^11
    with pytest.raises(AssertionError):
        X.norms32(table, "L2")
    with pytest.raises(AssertionError):
        X.scores64(table, table)
    X.norms32(table, "L2", bound=None)


def test_nonfinite_keys_rank_last_by_id_and_before_pads():
    """NaN and +inf keys are FLT_MAX: after every finite key, ties by id; -inf ranks first; all are returned before -1"""
    table, q, _ = _case(3, n_items=12, dim=4, n_q=1)
    table[2, 0] = 2.0 ** 64                                 # |t|^2 overflows: key +inf
    table[5] = np.nan
    table[9, 1] = -(2.0 ** 64)
    ids, dist = X.topk(q, table, "L2", 12, bound=None)
    assert ids[0, -3:].tolist() == [2, 5, 9]
    assert (dist[0, -3:] == FLT_MAX).all() and (dist[0, :-3] < FLT_MAX).all()
    rk = X.rank(np.repeat(q, 12, 0), table, "L2", np.arange(12), bound=None)
    assert np.array_equal(np.argsort(rk), ids[0]) and sorted(rk) == list(range(12))
    # exclusion leaves two eligible items, one of them FLT_MAX: it comes back before the pads
    ids, dist = X.topk(q, table, "L2", 4, exclude=[[j for j in range(12) if j not in (5, 7)]], bound=None)
    assert ids[0].tolist() == [7, 5, -1, -1]
    assert dist[0, 1] == FLT_MAX and (dist[0, 2:] == FLT_MAX).all()

    # IP: a query holding 2^126 twice makes <q, t> = 2^126 (t0 + t1) overflow for |t0 + t1| >= 4
    t = np.array([[3, 1], [-3, -1], [1, 1], [-2, -2], [2, 2], [0, 0]], np.float32)
    qq = np.full((1, 2), 2.0 ** 126, np.float32)
    s = X.scores64(qq, t, bound=None).to(torch.float32)
    assert s[0].tolist()[:2] == [float("inf"), float("-inf")]
    ids, dist = X.topk(qq, t, "IP", 6, bound=None)
    assert ids[0].tolist() == [0, 4, 2, 5, 1, 3]            # +inf first (key -inf), then finite, then -inf by id
    assert dist[0, 0] == np.inf and (dist[0, -2:] == -FLT_MAX).all()
    rk = X.rank(np.repeat(qq, 6, 0), t, "IP", np.arange(6), bound=None)
    assert np.array_equal(np.argsort(rk), ids[0])


def test_exclusion_and_candidates():
    table, q, _ = _case(4, n_items=40, dim=6, n_q=3)
    table[[3, 11, 20, 33]] = table[0]                        # a tie group 0, 3, 11, 20, 33
    qq = np.repeat(table[:1], 3, 0)
    ids, _ = X.topk(qq, table, "L2", 5, exclude=[[0, 3], [], list(range(40))])
    assert ids[0, :3].tolist() == [11, 20, 33]
    assert ids[1, :5].tolist() == [0, 3, 11, 20, 33]
    assert (ids[2] == -1).all()
    ids, _ = X.topk(qq, table, "L2", 5, candidates=[[33, 1, 20], list(range(40)), [2]])
    assert ids[0, :2].tolist() == [20, 33] and ids[0, 3:].tolist() == [-1, -1]
    assert ids[2].tolist() == [2, -1, -1, -1, -1]
    rk = X.rank(qq, table, "L2", [33, 33, 5], exclude=[[0, 3], [], [33]])
    assert rk[:2].tolist() == [2, 4]
