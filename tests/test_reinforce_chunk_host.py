"""Host-side checks of the chunked REINFORCE policy gradient: the chunk width rule of _policy_loss and the scratch size
of recnn_reinforce_scratch_floats.  No kernel is launched."""
from __future__ import annotations

import pytest

from recnn_b200 import _lib
from recnn_b200.nn.update import reinforce as RF


def dims(S, H, I):
    return _lib.DiscreteDims(S, H, I, 0)


def test_chunk_rule_single_chunk_up_to_the_budget():
    budget = RF._LOGITS_BUDGET_BYTES
    assert RF._chunk_items(1280, 5000) == 5000                      # bench.py's reinforce leg
    assert RF._chunk_items(4096, budget // (4096 * 4)) == budget // (4096 * 4)     # exactly at the budget
    assert RF._chunk_items(1, 1_000_000) == 1_000_000


@pytest.mark.parametrize("rows,items", [(4096, 262_144), (1280, 1_000_000), (163_840, 1_000_000), (4097, 65_536)])
def test_chunk_rule_above_the_budget(rows, items):
    budget = RF._LOGITS_BUDGET_BYTES
    assert rows * items * 4 > budget
    c = RF._chunk_items(rows, items)
    assert c % 128 == 0 and 128 <= c < items
    assert rows * c * 4 <= budget
    assert rows * (c + 128) * 4 > budget                          # the widest such multiple of 128


def test_chunk_rule_floor(monkeypatch):
    monkeypatch.setattr(RF, "_LOGITS_BUDGET_BYTES", 1000)
    assert RF._chunk_items(100, 100_000) == 128                   # 100 rows x 128 items exceed 1000 bytes: floor
    assert RF._chunk_items(100, 100) == 100                       # never wider than the vocabulary
    assert RF._chunk_items(2, 100) == 100                         # 800 bytes: fits


def test_chunked_scratch_does_not_grow_with_the_vocabulary():
    L = _lib.lib()
    for S, H, R, chunk in [(1290, 256, 4096, 512), (2570, 256, 163_840, 1536), (52, 64, 40, 128), (1290, 2048, 1280, 209_664)]:
        sizes = {L.recnn_reinforce_scratch_floats(dims(S, H, I), R, chunk) for I in (chunk + 1, 10_000 + chunk, 10**6)}
        assert len(sizes) == 1, (S, H, R, chunk, sizes)
        size = sizes.pop()
        assert size >= R * (S + 2 * H + chunk)
        # state image + two hidden buffers + one chunk + row statistics + the weight-gradient partials (+ alignment)
        assert size < R * (S + 3 + 2 * H + chunk + 8) + 2 * (chunk + 64 * 1024) * (H + 1) + 4096


@pytest.mark.parametrize("S,H,I,R", [(13, 16, 37, 6), (52, 64, 1000, 40), (1290, 256, 5000, 320), (1290, 2048, 5000, 1280),
                                     (1290, 256, 262_144, 4096)])
def test_single_chunk_scratch_fits_the_existing_query(S, H, I, R):
    L = _lib.lib()
    d = dims(S, H, I)
    single = L.recnn_reinforce_scratch_floats(d, R, I)
    assert 0 < single <= L.recnn_discrete_scratch_floats(d, R, 1)
    assert single >= R * I                                        # the whole logits matrix
    if I > 128:
        assert L.recnn_reinforce_scratch_floats(d, R, 128) < single


def test_scratch_query_rejects_bad_chunks():
    L = _lib.lib()
    d = dims(52, 64, 1000)
    for bad in (0, -128, 100, 129, 1024, 1001):
        assert L.recnn_reinforce_scratch_floats(d, 40, bad) == 0, bad
    assert L.recnn_reinforce_scratch_floats(d, 40, 896) > 0
    assert L.recnn_reinforce_scratch_floats(d, 0, 128) == 0
