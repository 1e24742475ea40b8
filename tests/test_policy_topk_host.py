"""Host-side checks of the REINFORCE policy's top-k: the C symbols, the workspace query, the refusals of
DiscreteActor.topk before any device work, and the float64 restatement (tests/_policy_topk_oracle.py) against a numpy
lexsort and against its own sharded merge.  No kernel is launched."""
from __future__ import annotations

import os
import re

import numpy as np
import pytest
import torch

import recnn_b200
from recnn_b200 import _lib
from recnn_b200 import dist as D
from tests import _policy_topk_oracle as TK

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW_SYMBOLS = ("recnn_discrete_topk_workspace_bytes", "recnn_discrete_topk", "recnn_vocab_topk_record_floats",
               "recnn_discrete_shard_topk", "recnn_discrete_shard_topk_finish")


def test_new_symbols_in_header_library_and_ctypes_table():
    with open(os.path.join(ROOT, "include", "recnn_b200.h")) as fh:
        declared = set(re.findall(r"RECNN_API\s+[\w\s\*]+?\b(recnn_\w+)\s*\(", fh.read()))
    L = _lib.lib()
    for name in NEW_SYMBOLS:
        assert name in declared and name in _lib.SIGNATURES
        assert getattr(L, name) is not None
    assert declared <= set(_lib.SIGNATURES), sorted(declared - set(_lib.SIGNATURES))
    assert L.recnn_b200_abi_version() == 3


def test_workspace_is_flat_in_the_vocabulary_when_chunked():
    L = _lib.lib()
    for S, H, N, k, chunk in [(2570, 256, 2048, 64, 131072), (37, 32, 33, 10, 128), (52, 64, 1, 1, 1 << 19)]:
        sizes = {L.recnn_discrete_topk_workspace_bytes(_lib.DiscreteDims(S, H, items, 0), N, k, chunk)
                 for items in (chunk + 1, 1 << 20, 8_000_003)}
        assert len(sizes) == 1 and sizes.pop() > 0, (S, N, chunk)
        ws = L.recnn_discrete_topk_workspace_bytes(_lib.DiscreteDims(S, H, 1 << 20, 0), N, k, chunk)
        # the state image, the hidden layer, one logits chunk, two row vectors and the [N, splits <= 31, k] lists
        assert ws < N * (S + 4 + H + chunk + 2) * 4 + N * 33 * k * 8 + 16 * 256
    d = _lib.DiscreteDims(52, 64, 1003, 0)
    assert L.recnn_discrete_topk_workspace_bytes(d, 40, 10, 1003) > 0
    assert L.recnn_discrete_topk_workspace_bytes(d, 40, 64, 128) > 0
    for n, k, chunk in [(40, 0, 1003), (40, 65, 1003), (40, 10, 100), (40, 10, 1004), (40, 10, 1024), (40, 10, 0),
                        (0, 10, 1003)]:
        assert L.recnn_discrete_topk_workspace_bytes(d, n, k, chunk) == 0, (n, k, chunk)
    assert L.recnn_vocab_topk_record_floats(40, 10) == 4 + 22 * 40
    assert L.recnn_vocab_topk_record_floats(40, 65) == 0


def test_python_refusals_happen_before_device_work():
    L = _lib.lib()
    torch.manual_seed(0)
    m = recnn_b200.nn.DiscreteActor(6, 10, 8)
    st = torch.zeros(3, 6)
    k0 = L.recnn_b200_launch_count()
    for k in (0, 11, 65, 2.0, True, None):
        with pytest.raises(ValueError, match="k must be"):
            m.topk(st, k)
    with pytest.raises(ValueError, match="state"):
        m.topk(torch.zeros(3, 5), 2)
    for ex in (torch.zeros(3, 2), torch.zeros(2, 2, dtype=torch.int64), torch.zeros(3, 257, dtype=torch.int64),
               torch.zeros(3, dtype=torch.int64), torch.zeros(3, 2, dtype=torch.bool), [[1, 2]] * 3):
        with pytest.raises(ValueError, match="exclude"):
            m.topk(st, 2, exclude=ex)
    with pytest.raises(_lib.RecnnError, match="CUDA only"):
        m.topk(st, 2, exclude=torch.zeros(3, 256, dtype=torch.int64))
    assert L.recnn_b200_launch_count() == k0


def _logits(seed, n, items, ties=False):
    rng = np.random.default_rng(seed)
    z = rng.normal(0, 2, (n, items))
    if ties:
        z = np.round(z, 1)                    # many exact ties
    return z


@pytest.mark.parametrize("ties", [False, True], ids=["distinct", "ties"])
def test_oracle_agrees_with_a_lexsort(ties):
    z = _logits(1, 30, 203, ties)
    for k in (1, 10, 64, 203):
        v, ids = TK.topk(z, k)
        for r in range(z.shape[0]):
            want = np.lexsort((np.arange(z.shape[1]), -z[r]))[:k]
            assert np.array_equal(ids[r], want)
        p = np.exp(z - z.max(1, keepdims=True))
        p /= p.sum(1, keepdims=True)
        np.testing.assert_allclose(v, np.take_along_axis(p, ids, 1), rtol=1e-12)


def test_oracle_exclusions_stay_in_the_normaliser():
    z = _logits(2, 12, 50, True)
    rng = np.random.default_rng(3)
    ex = rng.integers(-1, 50, (12, 30))
    ex[0] = -1
    v, ids = TK.topk(z, 30, ex)
    p = np.exp(z - z.max(1, keepdims=True))
    p /= p.sum(1, keepdims=True)
    for r in range(12):
        keep = np.setdiff1d(np.arange(50), ex[r])
        order = keep[np.lexsort((keep, -z[r, keep]))][:30]
        assert np.array_equal(ids[r, :len(order)], order)
        assert (ids[r, len(order):] == -1).all() and (v[r, len(order):] == 0).all()
        np.testing.assert_allclose(v[r, :len(order)], p[r, order], rtol=1e-12)


@pytest.mark.parametrize("world", [1, 2, 3, 8])
def test_oracle_sharded_merge_equals_the_unsharded_ranking(world):
    """1,003 and 100 items (13 per rank at W = 8: k = 64 exceeds every block), ties across the shard edges."""
    for items in (1003, 100):
        z = _logits(world, 25, items, True)
        edges = sorted({e for lo, hi in TK.item_plan(items, world) for e in (lo - 1, lo, hi - 1) if 0 <= e < items})
        z[:, edges] = 9.0
        ex = np.full((25, 3), -1)
        ex[:, 0] = edges[-1]
        for k in (1, 10, 64):
            for e in (None, ex):
                v1, i1 = TK.topk(z, k, e)
                vw, iw = TK.shard_topk(z, k, world, e)
                assert np.array_equal(iw, i1)
                np.testing.assert_allclose(vw, v1, rtol=1e-12)
        assert TK.item_plan(items, world) == [D.vocab_shard(items, q, world) for q in range(world)]
