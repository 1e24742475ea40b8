"""Host-side checks of diversified re-ranking: the entry point in the header, the library and the ctypes table; the
refusals of the C entry point and of ``diversify`` before any device work; and the float64 restatement
(tests/_diversify_oracle.py) against brute force on small pools -- MMR by its formula, the DPP's greedy choice as the
argmax of log det L over S + {i} and its stopping rule.  No kernel is launched."""
from __future__ import annotations

import os
import re

import numpy as np
import pytest
import torch

from recnn_b200 import _lib
from recnn_b200.utils import diversify
from tests import _diversify_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_symbol_in_header_library_and_ctypes_table():
    with open(os.path.join(ROOT, "include", "recnn_b200.h")) as fh:
        text = fh.read()
    declared = set(re.findall(r"RECNN_API\s+[\w\s\*]+?\b(recnn_\w+)\s*\(", text))
    assert "recnn_slate_diversify" in declared and "recnn_slate_diversify" in _lib.SIGNATURES
    assert declared <= set(_lib.SIGNATURES), sorted(declared - set(_lib.SIGNATURES))
    decl = re.search(r"RECNN_API int recnn_slate_diversify\((.*?)\);", text, re.S).group(1)
    assert "workspace" not in decl                    # nothing to size: the call allocates nothing
    assert len(decl.split(",")) == len(_lib.SIGNATURES["recnn_slate_diversify"][1])
    L = _lib.lib()
    assert getattr(L, "recnn_slate_diversify") is not None
    assert L.recnn_b200_abi_version() == 3


def test_c_refusals_before_device_work():
    L = _lib.lib()
    fake = 256                                        # never dereferenced: every call below is refused by its checks
    k0 = L.recnn_b200_launch_count()
    ok = [fake, fake, 4, 64, 10, fake, 100, 32, 0, 0.5, fake, fake, fake, fake, None]
    for i, bad in [(3, 0), (3, 257), (4, 0), (4, 65), (7, 0), (7, 1025), (8, 2), (8, -1), (9, -0.1), (9, 1.5),
                   (9, float("nan")), (6, 0), (2, -1), (0, None), (1, None), (5, None), (10, None), (11, None),
                   (12, None), (13, None)]:
        args = list(ok)
        args[i] = bad
        assert L.recnn_slate_diversify(*args) != 0, (i, bad)
    args = list(ok)
    args[3], args[4] = 8, 9                           # k > m
    assert L.recnn_slate_diversify(*args) != 0
    assert L.recnn_b200_launch_count() == k0


def test_module_refusals_happen_before_device_work():
    L = _lib.lib()
    k0 = L.recnn_b200_launch_count()
    ids = torch.tensor([[0, 1, -1], [2, 2, 3]])
    sc = torch.zeros(2, 3)
    table = torch.zeros(5, 4)
    for bad in (ids[0], ids.int(), ids.float(), ids.numpy(), torch.zeros(3, 0, dtype=torch.int64),
                torch.zeros(2, 257, dtype=torch.int64)):
        with pytest.raises(ValueError):
            diversify(bad, torch.zeros(tuple(bad.shape)) if torch.is_tensor(bad) else sc, table, 1)
    for bad in (sc.double(), sc.half(), sc[:, :2], sc[0], sc.numpy(), None):
        with pytest.raises(ValueError, match="scores"):
            diversify(ids, bad, table, 2)
    for bad_table in (table.double(), torch.zeros(5), torch.zeros(0, 4), torch.zeros(5, 0), torch.zeros(5, 1025),
                      None):
        with pytest.raises(ValueError, match="table"):
            diversify(ids, sc, bad_table, 2)
    for k in (0, 4, 2.0, True, None):
        with pytest.raises(ValueError, match="k"):
            diversify(ids, sc, table, k)
    with pytest.raises(ValueError, match="k"):
        diversify(torch.zeros(1, 100, dtype=torch.int64), torch.zeros(1, 100), table, 65)
    with pytest.raises(ValueError, match="method"):
        diversify(ids, sc, table, 2, method="xquad")
    for w in (-0.01, 1.01, float("nan"), True, "0.5", None):
        with pytest.raises(ValueError, match="weight"):
            diversify(ids, sc, table, 2, weight=w)
    if torch.cuda.is_available():
        with pytest.raises(ValueError, match="device"):
            diversify(ids, sc, table.cuda(), 2)
        with pytest.raises(ValueError, match="device"):
            diversify(ids.cuda(), sc, table.cuda(), 2)
    with pytest.raises(_lib.RecnnError, match="CUDA only"):       # no CPU path behind the kernel
        diversify(ids, sc, table, 2)
    assert L.recnn_b200_launch_count() == k0


# ----------------------------------------------------------------------------- the float64 restatement
def _pool(rng, m, D, n_items=12, repeat=True):
    table = rng.normal(0, 1, (n_items, D))
    table[3] = 0.0                                            # a zero vector
    ids = rng.integers(0, n_items, m)
    ids[rng.random(m) < 0.2] = -1
    if repeat and m >= 3:
        ids[m - 1] = ids[0] if ids[0] >= 0 else 5            # a repeated id
    return ids, rng.normal(0, 1, m), table


def _sim(a, b):
    na, nb = np.linalg.norm(a), np.linalg.norm(b)
    return 0.0 if na == 0 or nb == 0 else float(np.clip(a @ b / (na * nb), -1, 1))


@pytest.mark.parametrize("weight", [0.0, 0.3, 0.7, 1.0])
@pytest.mark.parametrize("seed", range(6))
def test_mmr_restatement_equals_the_formula(weight, seed):
    rng = np.random.default_rng(seed)
    m = 3 + seed
    ids, s, table = _pool(rng, m, 1 + seed)
    got, pos, gain = O.greedy(ids, s, table, m, "mmr", weight)
    picked = []
    for t in range(m):
        cand = [i for i in range(m) if ids[i] >= 0 and ids[i] not in [ids[j] for j in picked]]
        if not cand:
            assert got[t] == -1 and pos[t] == -1 and np.isnan(gain[t])
            continue
        obj = {i: weight * s[i] - (1 - weight) * (max(_sim(table[ids[i]], table[ids[j]]) for j in picked)
                                                  if picked else 0.0) for i in cand}
        best = max(obj.values())
        i = min((c for c in cand if obj[c] >= best - 1e-12), key=lambda c: (ids[c], c))
        assert pos[t] == i and got[t] == ids[i] and gain[t] == pytest.approx(obj[i], abs=1e-12)
        picked.append(i)
    assert len(set(got[got >= 0].tolist())) == (got >= 0).sum()          # a slate never repeats an id


def _logdet_L(X, s, alpha, cols):
    if not cols:
        return 0.0
    S = 0.5 * (1 + O.cosine_sim(X[cols]))
    q = np.exp(alpha * s[cols])
    sign, ld = np.linalg.slogdet(np.diag(q) @ S @ np.diag(q))
    return ld if sign > 0 else -np.inf


@pytest.mark.parametrize("weight", [0.0, 0.3, 0.7])
@pytest.mark.parametrize("D", [1, 2, 3, 8])
@pytest.mark.parametrize("seed", range(4))
def test_dpp_restatement_is_greedy_log_det_with_its_stopping_rule(weight, D, seed):
    rng = np.random.default_rng(100 * D + seed)
    m = 8
    ids, s, table = _pool(rng, m, D, repeat=seed % 2 == 0)
    X = np.zeros((m, D))
    X[ids >= 0] = table[ids[ids >= 0]]
    alpha = weight / (2 * (1 - weight))
    got, pos, gain = O.greedy(ids, s, table, m, "dpp", weight)
    picked = []
    for t in range(m):
        cand = [i for i in range(m) if ids[i] >= 0 and ids[i] not in [ids[j] for j in picked]]
        base = _logdet_L(X, s, alpha, picked)
        inc = {i: _logdet_L(X, s, alpha, picked + [i]) - base for i in cand}
        if pos[t] < 0:
            # stopped: nothing eligible, or the best increase has d^2 = det S[S+i] / det S[S] below eps
            if cand:
                best = max(inc.values())
                d2 = np.exp(best - 2 * alpha * s[max(inc, key=inc.get)])
                assert best == -np.inf or d2 < O.DPP_EPS * 1.001, (t, best, d2)
            assert (pos[t:] == -1).all() and (got[t:] == -1).all() and np.isnan(gain[t:]).all()
            break
        i = int(pos[t])
        assert i in cand and inc[i] >= max(inc.values()) - 1e-7, (t, i, inc)
        assert gain[t] == pytest.approx(inc[i], abs=1e-6)
        assert np.exp(inc[i] - 2 * alpha * s[i]) >= O.DPP_EPS * 0.999           # d^2 of the pick
        picked.append(i)
    assert (got >= 0).sum() <= D + 1                                             # rank S <= D + 1


def test_dpp_at_weight_one_and_on_orthogonal_rows_orders_by_score():
    rng = np.random.default_rng(5)
    m = 9
    ids = rng.permutation(20)[:m]
    s = rng.normal(0, 1, m)
    table = np.eye(20)
    want = ids[np.argsort(-s)]
    # one-hot rows: S = (I + 1 1^T) / 2, every unpicked column has the same d^2 at every step
    for w in (0.1, 0.4, 0.9):
        assert (O.greedy(ids, s, table, m, "dpp", w)[0] == want).all()
    assert (O.greedy(ids, s, table, m, "dpp", 0.0)[0] == np.sort(ids)).all()          # all tied: the smaller id
    got, pos, gain = O.greedy(ids, s, rng.normal(0, 1, (20, 2)), m, "dpp", 1.0)
    assert (got == want).all() and (gain == np.sort(s)[::-1]).all()


def test_ties_go_to_the_smaller_id_then_the_smaller_column():
    table = np.eye(6)
    ids = np.array([4, 2, 2, 5, -1, 1])
    s = np.array([1.0, 1.0, 1.0, 0.5, 3.0, 1.0])
    for method in ("mmr", "dpp"):
        got, pos, _ = O.greedy(ids, s, table, 4, method, 1.0)
        assert got.tolist() == [1, 2, 4, 5] and pos.tolist() == [5, 1, 0, 3]

