"""Host-side checks of the item-id critic: workspace and scratch sizes stay flat in num_items once the items are
chunked, the chunk rule is enforced, and the batch actions that have no item-id meaning are refused before any device
work."""
from __future__ import annotations

import ctypes

import pytest
import torch

import recnn_b200
from recnn_b200 import _lib
from recnn_b200.nn.update import _ids


def _dims(S, H, I):
    return _lib.Dims(S, I, H, 0), _lib.DiscreteDims(S, H, I, 0)


def test_workspace_does_not_grow_with_num_items():
    L = _lib.lib()
    sizes = []
    for I in (1 << 16, 1 << 18, 1 << 20):
        d, pd = _dims(2570, 256, I)
        ws = L.recnn_discrete_value_workspace_bytes(d, pd, 2048, 4096)
        sc = L.recnn_critic_action_term_scratch_floats(d, pd, 2048, 4096)
        assert ws > 0 and sc > 0
        sizes.append((ws, sc))
    assert len(set(sizes)) == 1
    d, pd = _dims(2570, 256, 1 << 20)
    # one [rows, chunk] chunk (with its `lead` pad columns) is the largest piece; nothing is [rows, num_items]
    assert sizes[0][0] < 2048 * (4096 + 4) * 4 + 2048 * (2 * 2572 + 16 * 256) * 4 + (32 << 20)
    assert L.recnn_discrete_value_workspace_bytes(d, pd, 2048, 1 << 20) > 2048 * (1 << 20) * 4    # single chunk


def test_chunk_rule_and_dims_are_checked():
    L = _lib.lib()
    d, pd = _dims(1290, 256, 5000)
    assert L.recnn_discrete_value_workspace_bytes(d, pd, 64, 100) == 0          # not a multiple of 128
    assert L.recnn_discrete_value_workspace_bytes(d, pd, 64, 5120) == 0         # wider than num_items
    assert L.recnn_discrete_value_workspace_bytes(d, pd, 64, 5000) > 0
    assert L.recnn_critic_action_term_scratch_floats(d, None, 64, 1280) > 0    # dense source: no policy buffers
    bad = _lib.DiscreteDims(1290, 256, 4999, 0)
    assert L.recnn_discrete_value_workspace_bytes(d, bad, 64, 128) == 0
    assert L.recnn_sizeof_discrete_value_args() == ctypes.sizeof(_lib.DiscreteValueArgs)


def test_action_kinds():
    assert _ids.is_item_ids(torch.tensor([3, 1, 4]))
    assert _ids.is_item_ids(torch.tensor([3, 1, 4], dtype=torch.int32))
    assert not _ids.is_item_ids(torch.zeros(3, 7))
    with pytest.raises(ValueError):
        _ids.is_item_ids(torch.zeros(3))                         # float [N]
    with pytest.raises(ValueError):
        _ids.is_item_ids(torch.zeros(3, 7, dtype=torch.int64))    # integer matrix


def test_update_steps_without_an_item_id_mode_refuse_ids():
    batch = {"state": torch.zeros(4, 6), "next_state": torch.zeros(4, 6), "action": torch.tensor([0, 1, 2, 1]),
             "reward": torch.zeros(4), "done": torch.zeros(4)}
    with pytest.raises(ValueError):
        recnn_b200.nn.td3_update(batch, {}, {}, {}, learn=True)
    with pytest.raises(ValueError):
        recnn_b200.nn.ddpg_update(batch, {}, {}, {}, learn=True)
    with pytest.raises(ValueError):
        recnn_b200.nn.value_update(dict(batch, action=torch.zeros(4)), {}, {}, {}, learn=True)
    actor_nets = {"target_policy_net": recnn_b200.nn.Actor(6, 3, 8)}
    with pytest.raises(ValueError):
        recnn_b200.nn.value_update(batch, {}, actor_nets, {}, learn=True)
