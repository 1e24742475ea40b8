"""Host-side checks of serving through the DDPG / TD3 critic: the entry points in the header, the library and the ctypes
table; the all-items workspace bound; the refusals of Critic.topk / Critic.rank before any device work; and the float64
restatement against brute-force numpy orderings.  No kernel is launched."""
from __future__ import annotations

import os
import re

import numpy as np
import pytest
import torch

import recnn_b200
from recnn_b200 import _lib
from recnn_b200.data import ItemSets
from tests import _critic_serve_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW_SYMBOLS = ("recnn_critic_serve_workspace_bytes", "recnn_critic_topk", "recnn_critic_rank")


def test_new_symbols_in_header_library_and_ctypes_table():
    with open(os.path.join(ROOT, "include", "recnn_b200.h")) as fh:
        declared = set(re.findall(r"RECNN_API\s+[\w\s\*]+?\b(recnn_\w+)\s*\(", fh.read()))
    L = _lib.lib()
    for name in NEW_SYMBOLS:
        assert name in declared and name in _lib.SIGNATURES, name
        assert getattr(L, name) is not None
    assert declared <= set(_lib.SIGNATURES), sorted(declared - set(_lib.SIGNATURES))
    assert not any(name.endswith("_sets") for name in declared if name.startswith("recnn_critic_"))
    assert L.recnn_b200_abi_version() == 3


def test_all_items_workspace_does_not_grow_with_the_table():
    L = _lib.lib()
    d = _lib.Dims(1290, 128, 256, 0)
    for n, k, chunk in [(64, 10, 0), (2048, 64, 0), (2048, 0, 0), (128, 10, 1000), (16384, 1, 0)]:
        a = L.recnn_critic_serve_workspace_bytes(d, n, 0, 131072, k, chunk)
        b = L.recnn_critic_serve_workspace_bytes(d, n, 0, 262144, k, chunk)
        assert a == b > 0, (n, k, chunk)
        # O(rows (S + H + k)) plus one block of pair buffers: far below one [n, n_items] score matrix
        assert a < n * (1292 + 256 + 16 * max(k, 1)) * 4 + (64 << 20), (n, k, a)
    # a candidate call's block is sized by its candidates, not by the table
    assert (L.recnn_critic_serve_workspace_bytes(d, 2048, 1024, 1 << 20, 10, 0)
            == L.recnn_critic_serve_workspace_bytes(d, 2048, 1024, 4096, 10, 0))
    assert L.recnn_critic_serve_workspace_bytes(d, 0, 0, 100, 10, 0) == 0
    assert L.recnn_critic_serve_workspace_bytes(d, 4, 0, 100, 65, 0) == 0
    assert L.recnn_critic_serve_workspace_bytes(d, 4, 0, 100, 10, -1) == 0


def test_c_refusals_before_device_work():
    L = _lib.lib()
    d = _lib.Dims(6, 4, 8, 0)
    fake = 256                                  # never dereferenced: every call below is refused by its checks
    k0 = L.recnn_b200_launch_count()
    ws = 1 << 30
    assert L.recnn_critic_topk(d, fake, fake, 4, fake, 100, None, 0, 0, None, 0, None, 0, None, 0, fake, fake, fake,
                               fake, ws, None) != 0                                       # k = 0
    assert L.recnn_critic_topk(d, fake, fake, 4, fake, 100, None, 0, 65, None, 0, None, 0, None, 0, fake, fake, fake,
                               fake, ws, None) != 0                                       # k > 64
    assert L.recnn_critic_topk(d, fake, fake, 4, fake, 100, None, 5, 3, None, 0, None, 0, None, 0, fake, fake, fake,
                               fake, ws, None) != 0                                       # n_candidates without a list
    assert L.recnn_critic_topk(d, fake, fake, 4, fake, 100, None, 0, 3, None, 0, None, 0, None, 0, fake, fake, fake,
                               fake, 16, None) != 0                                       # workspace
    assert L.recnn_critic_rank(d, fake, fake, 4, fake, 100, None, 0, None, None, 0, None, 0, None, 0, fake, fake,
                               fake, ws, None) != 0                                       # no target
    assert L.recnn_critic_rank(d, fake, fake, 4, fake, 100, None, 0, fake, None, 0, fake, 3, None, 0, fake, fake,
                               fake, ws, None) != 0                                       # 3 sets for 4 rows, no map
    assert L.recnn_b200_launch_count() == k0


def test_module_refusals_happen_before_device_work():
    L = _lib.lib()
    torch.manual_seed(0)
    c = recnn_b200.nn.Critic(6, 4, 8)                    # on the CPU: a refusal must come before the device check
    st, table = torch.zeros(3, 6), torch.zeros(20, 4)
    cand = torch.tensor([[1, 2], [3, 4], [5, -1]])
    tgt = torch.tensor([1, 2, 3])
    sets = ItemSets.from_lists([[1], [2], [3]])
    k0 = L.recnn_b200_launch_count()
    for k in (0, 65, 2.0, True):
        with pytest.raises(ValueError, match="k must"):
            c.topk(st, k, table)
    calls = [lambda **kw: c.topk(st, 2, **kw), lambda **kw: c.rank(st, tgt, **kw)]
    for bad_state in (torch.zeros(3, 5), torch.zeros(6), torch.zeros(3, 6, dtype=torch.int64)):
        with pytest.raises(ValueError, match="state"):
            c.topk(bad_state, 2, table)
        with pytest.raises(ValueError, match="state"):
            c.rank(bad_state, tgt, table)
    for call in calls:
        for bad_table in (torch.zeros(20, 4, dtype=torch.float64), torch.zeros(20), np.zeros((20, 4), np.float32),
                          torch.zeros(0, 4)):
            with pytest.raises(ValueError, match="items"):
                call(items=bad_table)
        with pytest.raises(ValueError, match="action_dim"):
            call(items=torch.zeros(20, 5))
        for bad_cand in (torch.zeros(3, 2), torch.zeros(2, 2, dtype=torch.int64), torch.zeros(3, dtype=torch.int64),
                         torch.zeros(3, 0, dtype=torch.int64), torch.zeros(3, 2, dtype=torch.bool)):
            with pytest.raises(ValueError, match="candidates"):
                call(items=table, candidates=bad_cand)
        with pytest.raises(ValueError, match="ItemSets"):
            call(items=table, exclude=torch.zeros(3, 2, dtype=torch.int64))
        with pytest.raises(ValueError, match="exclude_rows"):
            call(items=table, exclude_rows=torch.zeros(3, dtype=torch.int64))
        with pytest.raises(ValueError, match="sets"):
            call(items=table, exclude=ItemSets.from_lists([[1], [2]]))
        with pytest.raises(ValueError, match="chunk"):
            call(items=table, chunk=-1)
        with pytest.raises(_lib.RecnnError, match="CUDA"):          # every argument is fine: only the device is not
            call(items=table, candidates=cand, exclude=sets)
    for bad_t in (torch.zeros(3), torch.tensor([1, 2]), [1, 2, 3]):
        with pytest.raises(ValueError, match="target"):
            c.rank(st, bad_t, table)
    assert L.recnn_b200_launch_count() == k0


def test_split_form_equals_the_plain_forward():
    rng = np.random.default_rng(0)
    S, A, H, I, N = 9, 5, 7, 40, 6
    p = {"w1": rng.normal(0, .3, (H, S + A)), "b1": rng.normal(0, .3, H), "w2": rng.normal(0, .3, (H, H)),
         "b2": rng.normal(0, .3, H), "w3": rng.normal(0, .3, (1, H)), "b3": rng.normal(0, .3, 1)}
    state, table = rng.normal(0, 1, (N, S)), rng.normal(0, 1, (I, A))
    ids = rng.integers(-1, I, (N, 12))
    a, b = O.q_pairs(p, state, table, ids, rows_per_step=4), O.q_pairs_direct(p, state, table, ids)
    assert np.array_equal(np.isnan(a), ids < 0)
    np.testing.assert_allclose(a[ids >= 0], b[ids >= 0], rtol=1e-12, atol=1e-12)


def _brute(q_row, ids_row, ex):
    """argsort of (-q, id) over the eligible columns: the full order of one row."""
    keep = np.array([i >= 0 and i not in ex for i in ids_row], bool)
    qs, ii = np.asarray(q_row)[keep], np.asarray(ids_row)[keep]
    o = np.lexsort((ii, -qs))
    return qs[o], ii[o]


def test_restatement_against_brute_force_orderings():
    rng = np.random.default_rng(1)
    N, I, M = 40, 30, 12
    for trial in range(4):
        q_all = rng.integers(0, 6, (N, I)).astype(np.float64) / 4      # many exact ties
        ids = np.stack([rng.permutation(I)[:M] for _ in range(N)])
        ids[rng.random((N, M)) < 0.2] = -1                              # padding
        q = np.take_along_axis(q_all, np.where(ids >= 0, ids, 0), 1)
        q[ids < 0] = np.nan
        exclude = [sorted(set(rng.integers(0, I, rng.integers(0, 8)).tolist())) for _ in range(N)]
        exclude[0] = sorted(set(ids[0][ids[0] >= 0].tolist()))          # a set covering every candidate
        target = rng.integers(0, I, N)
        for k in (1, 5, 12, 20):
            vals, got = O.topk(q, ids, k, exclude)
            for r in range(N):
                bq, bi = _brute(q[r], ids[r], set(exclude[r]))
                m = min(k, bi.size)
                assert np.array_equal(got[r, :m], bi[:m]) and np.array_equal(vals[r, :m], bq[:m])
                assert (got[r, m:] == -1).all() and (vals[r, m:] == -O.FLT_MAX).all()
            assert (got[0] == -1).all()
        rk = O.rank(q, ids, target, exclude)
        rk_all = O.rank(q_all, O.all_ids(N, I), target, exclude)
        for r in range(N):
            ex = set(exclude[r]) - {int(target[r])}
            bq, bi = _brute(q[r], ids[r], ex)
            hit = np.nonzero(bi == target[r])[0]
            assert rk[r] == (hit[0] if hit.size else bi.size), (trial, r)    # absent target: the eligible count
            _, ai = _brute(q_all[r], np.arange(I), ex)
            assert rk_all[r] == np.nonzero(ai == target[r])[0][0]
            if hit.size and hit[0] < 20:                                 # the rank is the position in topk
                _, t20 = O.topk(q[r:r + 1], ids[r:r + 1], 20, [sorted(ex)])
                assert t20[0, rk[r]] == target[r]
