"""recnn.nn.update.misc equivalents (recnn/nn/update/misc.py:6-55)."""
from __future__ import annotations

import torch

from ... import _lib
from ... import utils
from ._engine import get_engine
from . import _ids


def temporal_difference(reward, done, gamma, target):
    """reward + (1 - done) * gamma * target   (misc.py:6-7).  Plain tensor algebra kept for
    API parity; inside the update step it is fused into the critic-head kernel."""
    return reward + (1.0 - done) * gamma * target


def value_update(batch, params, nets, optimizer, device=torch.device("cpu"), debug=None,
                 writer=utils.DummyWriter(), learn=False, step=-1):
    """DDPG critic step on its own (misc.py:10-55).  Returns the value loss as a 0-dim tensor
    (the reference returns the loss tensor, not a float).

    With a DiscreteActor target policy, ``batch["action"]`` may be an integer tensor of item ids [N] instead of the
    dense one-hot [N, num_items]: the same update then runs without any [N, num_items] buffer (recnn_b200/nn/update/
    _ids.py), which is what makes a million-item critic fit on one GPU."""
    if _ids.is_item_ids(batch["action"]):
        if not _ids._is_discrete(nets["target_policy_net"]):
            raise ValueError("item-id actions need a DiscreteActor target policy (nets['target_policy_net'])")
        return torch.tensor(_ids.get_ids_step(nets, device).run(batch, params, nets, optimizer, learn, debug))
    if nets.get("value_net") is not None and "_recnn_vp" in nets["value_net"].__dict__:
        raise RuntimeError("a vocabulary-parallel critic (enable_vocab_parallel) is trained on item-id batch actions only")
    eng = get_engine(_lib.ALGO_DDPG, nets, device)
    vals = eng.value_only(batch, params, nets, optimizer, learn, debug)
    return torch.tensor(vals[0])
