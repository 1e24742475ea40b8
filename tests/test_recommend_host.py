"""Host-side checks of serving with exclusion sets: ItemSets construction against numpy, the refusals of
DiscreteActor.topk / ItemIndex.search / DeviceFrameFeed.user_states before any device work, the new C symbols and
workspace sizes that do not depend on the sets.  No kernel is launched."""
from __future__ import annotations

import os
import re

import numpy as np
import pytest
import torch

import recnn_b200
from recnn_b200 import _lib
from recnn_b200.data import ItemSets, HistoryCSR

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW_SYMBOLS = ("recnn_discrete_topk_sets", "recnn_discrete_shard_topk_sets", "recnn_retrieve_topk_sets",
               "recnn_user_states")


def _random_lists(seed, n_sets, max_len, items):
    rng = np.random.default_rng(seed)
    return [rng.integers(0, items, rng.integers(0, max_len + 1)) for _ in range(n_sets)]


def test_new_symbols_in_header_library_and_ctypes_table():
    with open(os.path.join(ROOT, "include", "recnn_b200.h")) as fh:
        declared = set(re.findall(r"RECNN_API\s+[\w\s\*]+?\b(recnn_\w+)\s*\(", fh.read()))
    L = _lib.lib()
    for name in NEW_SYMBOLS:
        assert name in declared and name in _lib.SIGNATURES
        assert getattr(L, name) is not None
    assert declared <= set(_lib.SIGNATURES), sorted(declared - set(_lib.SIGNATURES))


@pytest.mark.parametrize("unique", [False, True])
def test_item_sets_sort_within_sets_against_numpy(unique):
    lists = _random_lists(0, 40, 30, 12)                 # few items: many duplicates
    lists[3] = np.zeros(0, dtype=np.int64)
    s = ItemSets.from_lists(lists, unique=unique)
    assert len(s) == 40 and s.ids.dtype == torch.int64 and s.offsets.dtype == torch.int64
    assert int(s.offsets[0]) == 0 and int(s.offsets[-1]) == s.ids.numel()
    for i, x in enumerate(lists):
        want = np.unique(x) if unique else np.sort(x)
        assert np.array_equal(s.set(i).numpy(), want), i
    flat = np.concatenate(lists)
    offs = np.concatenate([[0], np.cumsum([len(x) for x in lists])])
    t = ItemSets(torch.from_numpy(flat), torch.from_numpy(offs), unique=unique)
    assert torch.equal(t.ids, s.ids) and torch.equal(t.offsets, s.offsets)


def test_item_sets_refuse_bad_offsets_and_types():
    ids = torch.arange(5)
    for offs in ([1, 5], [0, 4], [0, 3, 2, 5], [0, 6], []):
        with pytest.raises(ValueError, match="offsets"):
            ItemSets(ids, torch.tensor(offs, dtype=torch.int64))
    with pytest.raises(ValueError, match="ids"):
        ItemSets(torch.zeros(5), torch.tensor([0, 5]))
    with pytest.raises(ValueError, match="ids"):
        ItemSets(torch.zeros(5, 1, dtype=torch.int64), torch.tensor([0, 5]))
    empty = ItemSets.from_lists([])
    assert len(empty) == 0 and empty.ids.numel() == 0


def test_python_refusals_happen_before_device_work():
    L = _lib.lib()
    torch.manual_seed(0)
    m = recnn_b200.nn.DiscreteActor(6, 10, 8)
    st = torch.zeros(3, 6)
    sets = ItemSets.from_lists([[1], [2, 3]])
    k0 = L.recnn_b200_launch_count()
    with pytest.raises(ValueError, match="sets but the call has 3 rows"):
        m.topk(st, 2, exclude=sets)
    for rows in (torch.zeros(2, dtype=torch.int64), torch.zeros(3), torch.zeros(3, 1, dtype=torch.int64)):
        with pytest.raises(ValueError, match="exclude_rows"):
            m.topk(st, 2, exclude=sets, exclude_rows=rows)
    with pytest.raises(ValueError, match="exclude_rows"):
        m.topk(st, 2, exclude=torch.zeros(3, 2, dtype=torch.int64), exclude_rows=torch.zeros(3, dtype=torch.int64))
    with pytest.raises(_lib.RecnnError, match="CUDA only"):
        m.topk(st, 2, exclude=sets, exclude_rows=torch.tensor([0, -1, 1]))
    assert L.recnn_b200_launch_count() == k0


def test_history_tables_refuse_short_users_on_the_host():
    csr = HistoryCSR([7, 8], [[1, 2, 3], [4, 5]], [[1, 1, 1], [2, 2]], frame_size=3)
    assert csr.check_positions([0]).tolist() == [0]
    with pytest.raises(ValueError, match="fewer than frame_size"):
        csr.check_positions([0, 1])


def test_workspace_does_not_depend_on_the_sets():
    """The *_sets calls take recnn_discrete_topk_workspace_bytes / recnn_retrieve_workspace_bytes, whose arguments
    name no table: the same bytes for a set of 1 id or of 1M ids; the dense form's sorted copy is bounded by N * 256."""
    L = _lib.lib()
    d = _lib.DiscreteDims(2570, 256, 1 << 20, 0)
    for n, k, chunk in [(2048, 64, 131072), (1, 10, 1 << 20), (16384, 10, 8192)]:
        ws = L.recnn_discrete_topk_workspace_bytes(d, n, k, chunk)
        assert 0 < ws < n * (2572 + 256 + chunk + 2) * 4 + n * 33 * k * 8 + n * 256 * 8 + 16 * 256
    assert L.recnn_retrieve_workspace_bytes(2048, 1 << 20, 10) > 0
