"""The bit-exact serving restatement (tests/_exact_serving.py) on the host: its builders refuse nets outside the
exact bounds, its orders agree with a sorted() brute force and with the float64 oracles on tie-free cases, and the
exact-pi rule holds in a numpy fp32 replay of the device's reduction."""
from __future__ import annotations

import numpy as np
import pytest

from tests import _critic_serve_oracle as CO
from tests import _exact_serving as X
from tests import _policy_topk_oracle as TK


def _policy(seed=0, S=20, H=16, I=300, N=12):
    rng = np.random.default_rng(seed)
    p = X.policy_params(rng, S, H, I)
    return p, X.policy_state(rng, N, S)


def test_builders_refuse_cases_outside_the_bounds():
    p, state = _policy()
    X.policy_logits(p, state)
    big = {k: v.copy() for k, v in p.items()}
    big["w1"][0, 0] = 2 ** 11 + 1                          # an operand TF32 does not hold
    with pytest.raises(AssertionError, match="exceeds 2"):
        X.policy_logits(big, state)
    frac = {k: v.copy() for k, v in p.items()}
    frac["w2"][3, 2] = 0.5
    with pytest.raises(AssertionError, match="not integer"):
        X.policy_logits(frac, state)
    wide = {k: v.copy() for k, v in p.items()}                 # h within 2^11, but sum |w2 h| reaches 2^24
    wide["w1"][:] = 0
    wide["b1"][:] = 2 ** 11
    wide["w2"][:] = 2 ** 11
    with pytest.raises(AssertionError, match="2\\^24"):
        X.policy_logits(wide, state)
    rng = np.random.default_rng(1)
    c = X.critic_params(rng, 9, 5, 8)
    st, tb = X.small_ints(rng, (3, 9)), X.small_ints(rng, (20, 5))
    X.critic_q(c, st, tb)
    with pytest.raises(AssertionError):
        X.critic_q(c, st * 4096, tb)


def _brute_topk(key, k, ok):
    out = np.full(k, -1)
    best = sorted((float(key[j]), j) for j in range(len(key)) if ok[j])[:k]
    out[:len(best)] = [j for _, j in best]
    return out


def test_orders_against_a_brute_force_with_ties_and_non_finite_logits():
    p, state = _policy(2)
    z = X.policy_logits(p, state)
    z[:, [3, 17, 200]] = -np.inf
    z[1, [5, 6]] = np.nan
    rng = np.random.default_rng(3)
    lists = [sorted(rng.choice(300, 40, replace=False).tolist()) for _ in range(len(z))]
    key = X.keys32(z).numpy()
    assert key.dtype == np.float32 and (key[:, 3] == X.FLT_MAX).all() and (key[1, 5] == X.FLT_MAX)
    ok = X.eligible(len(z), 300, lists)
    for k in (1, 17, 64):
        got = X.topk(z, k, lists)
        for r in range(len(z)):
            assert np.array_equal(got[r], _brute_topk(key[r], k, ok[r])), (k, r)
    tgt = rng.integers(0, 300, len(z))
    tgt[0] = 3
    got = X.rank(z, tgt, lists)
    for r, t in enumerate(tgt):
        okr = ok[r].copy()
        okr[t] = True                                        # a target is never excluded
        order = _brute_topk(key[r], 300, okr)
        assert got[r] == list(order).index(t), r


def test_orders_agree_with_the_float64_oracles_without_ties():
    rng = np.random.default_rng(4)
    z = rng.permutation(np.arange(-500, 500, dtype=np.float64))[:400].reshape(4, 100)      # distinct integers
    ex = np.stack([rng.choice(100, 10, replace=False) for _ in range(4)])
    for k in (1, 10, 64):
        assert np.array_equal(X.topk(z, k, ex), TK.topk(z, k, ex)[1])
    cols = np.stack([rng.permutation(100)[:30] for _ in range(4)])
    cols[:, ::4] = -1
    tgt = np.array([cols[0, 1], 7, cols[2, 3], 55])
    q_cols = z[np.arange(4)[:, None], np.maximum(cols, 0)]                # the oracle's Q per candidate column
    assert np.array_equal(X.topk(z, 12, ex, cols), CO.topk(q_cols, cols, 12, ex)[1])
    want = CO.rank(q_cols, cols, tgt, ex)
    assert np.array_equal(X.rank(z, tgt, [[x for x in e if x != t] for e, t in zip(ex, tgt)], cols), want)


def test_topk_splits_restatement():
    assert X.topk_splits(8, 40000) == 31
    assert X.topk_splits(40, 7000) == 7
    assert X.topk_splits(40, 1003) == 1 and X.topk_splits(70000, 300) == 1
    assert X.split_edges(40, 7000) == [i * 1000 for i in range(7)]
    assert X.split_edges(8, 1000, 256) == [0, 256, 512, 768]


def _replay(z, threads=256, chunk=None):
    """numpy fp32 replay of logit_stats_kernel / softmax_rows_kernel (np.exp for __expf: the exact-pi rows use only
    e^0 and e^d with d <= -128, where both give 1 and 0) and the chunk merge"""
    f = np.float32
    I = len(z)
    chunk = chunk or I
    Mr = Sr = None
    for c0 in range(0, I, chunk):
        w = z[c0:c0 + chunk].astype(f)
        ms, ss = [], []
        for t in range(threads):
            m, s = f(-np.inf), f(0)
            for x in w[t::threads]:
                if x > m:
                    s = f(s * np.exp(f(m - x))) + f(1)
                    m = x
                elif x != -np.inf:
                    s = f(s + np.exp(f(x - m)))
            ms.append(m)
            ss.append(s)
        M = max(ms)
        S = f(0)
        for m, s in zip(ms, ss):
            S = f(S + (f(0) if m == -np.inf else f(s * np.exp(f(m - M)))))
        if Mr is None:
            Mr, Sr = M, S
        else:
            Mn = max(Mr, M)
            Sr = f(0) if Mn == -np.inf else f(f(Sr * np.exp(f(Mr - Mn))) + f(S * np.exp(f(M - Mn))))
            Mr = Mn
    with np.errstate(over="ignore", under="ignore"):
        return np.array([f(np.exp(f(x - Mr)) / Sr) for x in z.astype(f)], f)


@pytest.mark.parametrize("chunk", [None, 128])
def test_exact_pi_rule_in_an_fp32_replay(chunk):
    rng = np.random.default_rng(6)
    z = rng.integers(-20, 20, 1003).astype(np.float64)
    z[:300:7] = -np.inf
    z[[0, 255, 256, 511, 640, 1002]] = 300.0
    with np.errstate(over="ignore", under="ignore"):
        ok, pi = X.exact_pi_rows(z[None, :])
        assert ok[0]
        assert np.array_equal(_replay(z, chunk=chunk).view(np.int32), pi[0].view(np.int32))
    assert pi[0, 0] == np.float32(1 / 6) and (pi[0, 1:255] == 0).all()
    z[3] = 299.0                                             # within 128 of the max: not an exact row
    assert not X.exact_pi_rows(z[None, :])[0][0]
