"""Drop-in for recnn.nn.update.ddpg_update (recnn/nn/update/ddpg.py:8-104)."""
from __future__ import annotations

import torch

from ... import _lib
from ... import utils
from ._engine import get_engine
from ._ids import reject_ids


def ddpg_update(batch, params, nets, optimizer, device=torch.device("cpu"), debug=None,
                writer=utils.DummyWriter(), learn=False, step=-1):
    """Same signature, defaults, side effects and return value as the reference:
    mutates the online nets (through the optimizers), the optimizer state and --
    on policy steps -- the target nets; returns ``{"value", "policy", "step"}``
    with Python floats.

    ``batch`` is either the reference's dense dict (state, action, reward,
    next_state, done) or the frame form produced by recnn_b200.data (items,
    ratings, done|sizes, table), in which case the embedding gather runs on the
    device as part of the step.  Optional ``batch["dropout_masks"]`` (six uint8
    [N,H] keep-masks in the reference's drop_layer call order) makes the step
    bit-reproducible; without it dropout uses an on-device Philox stream.

    ``device`` must be a CUDA device (the reference defaults to CPU; this
    implementation has no CPU path and raises instead of silently falling back).
    """
    if not learn and debug is None:
        # the reference fails the same way: debug["next_action"] = ... on None (misc.py:47)
        raise TypeError("'NoneType' object does not support item assignment")
    reject_ids(batch, "ddpg_update")
    eng = get_engine(_lib.ALGO_DDPG, nets, device)
    vals = eng.step(batch, params, nets, optimizer, learn, step, debug, "policy_step")
    losses = {"value": vals[0], "policy": vals[2], "step": step}
    utils.write_losses(writer, losses, kind="train" if learn else "test")
    return losses
