"""Drop-in for recnn.nn.update.td3_update (recnn/nn/update/td3.py:8-150)."""
from __future__ import annotations

import torch

from ... import _lib
from ... import utils
from ._engine import get_engine
from ._ids import reject_ids


def td3_update(batch, params, nets, optimizer, device=torch.device("cpu"), debug=None,
               writer=utils.DummyWriter(), learn=False, step=-1):
    """Same signature / side effects / return value as the reference
    (``{"value1", "value2", "policy", "step"}``).  Quirks kept: no clamp on the TD
    target, the target policy is never soft-updated, the actor gradient goes
    through value_net1 only.  ``batch["noise"]`` (the raw N(0, noise_std) draw,
    fp32 [N, A]) and ``batch["dropout_masks"]`` (eight masks) make the step
    bit-reproducible; otherwise both come from the on-device Philox stream (the
    reference draws the noise on the CPU generator, td3.py:74)."""
    if debug is None:
        debug = dict()           # td3.py:66-67
    reject_ids(batch, "td3_update")
    eng = get_engine(_lib.ALGO_TD3, nets, device)
    vals = eng.step(batch, params, nets, optimizer, learn, step, debug, "policy_update")
    losses = {"value1": vals[0], "value2": vals[1], "policy": vals[2], "step": step}
    utils.write_losses(writer, losses, kind="train" if learn else "test")
    return losses
