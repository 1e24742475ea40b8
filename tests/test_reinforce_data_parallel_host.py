"""Host-side checks of the data-parallel REINFORCE agent (no GPU): the new C symbols, the refusals of
enable_data_parallel, and float64 restatements of the row-sharded item-id critic step and of the row-offset draws."""
from __future__ import annotations

import ctypes
import re

import numpy as np
import pytest
import torch

import recnn_b200
from recnn_b200 import _lib
from recnn_b200 import build as _build
from recnn_b200 import dist as D
from oracle import reinforce_oracle as RO
from tests import _critic_vocab_oracle as CV
from tests import _philox as PH
from tests._discrete import PARAMS, critic_case
from tests._ranks import one_rank_cpu_group  # noqa: F401

NEW = ("recnn_categorical_sample_at", "recnn_discrete_value_dp_grad_floats", "recnn_discrete_value_dp_record_floats",
       "recnn_discrete_value_dp_workspace_bytes", "recnn_discrete_value_dp_begin", "recnn_discrete_value_dp_end")


def test_symbols_agree_between_header_library_and_ctypes():
    header = open(_build.ROOT + "/include/recnn_b200.h").read()
    lib = _lib.lib()
    for name in NEW:
        assert re.search(r"RECNN_API\s+\w+\s+%s\(" % name, header), name
        assert name in _lib.SIGNATURES, name
        assert hasattr(lib, name), name


def test_beta_args_probe_holds():
    lib = _lib.lib()
    assert lib.recnn_sizeof_beta_args() == ctypes.sizeof(_lib.BetaArgs)
    i = _lib._BETA_PROBE_FIELDS.index("n_rows_global")
    assert lib.recnn_offsetof_beta_args(i) == _lib.BetaArgs.n_rows_global.offset


def test_message_sizes_do_not_grow_with_the_vocabulary():
    lib = _lib.lib()
    S, H = 2570, 256
    for items in (5000, 1 << 20):
        d = _lib.Dims(S, items, H, 0)
        assert lib.recnn_discrete_value_dp_grad_floats(d) == H * ((S + 3) // 4 * 4 + H + 3) + 3
        assert lib.recnn_discrete_value_dp_record_floats(d, 130) == 4 + 132 + 130 * H


# ----------------------------------------------------------------------------- refusals
def _cpu_agent():
    torch.manual_seed(0)
    return recnn_b200.nn.Reinforce(recnn_b200.nn.DiscreteActor(8, 20, 16), recnn_b200.nn.Critic(8, 20, 16))


def test_refusals_happen_before_any_device_work(one_rank_cpu_group):
    agent = _cpu_agent()
    agent.nets["value_net"].__dict__["_recnn_vp"] = object()
    with pytest.raises(RuntimeError, match="do not combine"):
        D.enable_data_parallel(agent)
    agent = _cpu_agent()
    agent.optimizers["value_optimizer"] = torch.optim.Adam(agent.nets["value_net"].parameters())
    for p in agent.nets["value_net"].parameters():
        p.grad = torch.zeros_like(p)
    agent.optimizers["value_optimizer"].step()
    with pytest.raises(RuntimeError, match="already holds state"):
        D.enable_data_parallel(agent)
    ddpg = recnn_b200.nn.DDPG(recnn_b200.nn.Actor(8, 4, 16), recnn_b200.nn.Critic(8, 4, 16))
    with pytest.raises(TypeError, match="DiscreteActor"):
        D.enable_data_parallel(ddpg, beta=recnn_b200.nn.Beta(8, 4))
    # nothing was attached by a refused call
    assert all("_recnn_rows" not in n.__dict__ for n in agent.nets.values())
    # and the reverse: a data-parallel agent is not sharded over the vocabulary
    agent = _cpu_agent()
    D.data_parallel_in_place(dict(agent.nets), D.RowParallel(None, 0, 1, None))
    with pytest.raises(RuntimeError, match="do not combine"):
        D.enable_vocab_parallel(agent)


# ----------------------------------------------------------------------------- float64 restatements
def _dp_value_step(nets, batch, params, masks, world):
    """The row-sharded critic step: each rank's replicated gradient over its rows (MSE over 1 / N_global), summed over
    the ranks in rank order, and the action block scattered from the gathered dz1 rows in ascending (id, row) order."""
    p, tp, tv = nets["value_net"], nets["target_policy_net"], nets["target_value_net"]
    S = tp["w1"].shape[1]
    a_all = np.asarray(batch["action"])
    n = len(a_all)
    items = tp["w2"].shape[0]
    total, loss, rows = None, 0.0, []
    for r in range(world):
        lo, hi = D.shard_rows(n, r, world)
        b = {k: np.asarray(v)[lo:hi] for k, v in batch.items()}
        x, x2 = (np.asarray(b[k], np.float64) for k in ("state", "next_state"))
        a = b["action"]
        probs, _ = RO.discrete_forward(tp, x2)
        q2, _ = CV._critic_tail(tv, S, x2, probs @ np.asarray(tv["w1"], np.float64)[:, S:].T, None)
        y = CV._td(b, q2, params)
        add = np.asarray(p["w1"], np.float64)[:, S + a].T
        m = None if masks is None else [mm[lo:hi] for mm in masks]
        q, cache = CV._critic_tail(p, S, x, add, m)
        diff = q - y
        g, dz1 = CV._backward(S, x, cache, 2.0 * diff / n)
        loss += float((diff * diff).sum()) / n
        total = g if total is None else {k: total[k] + g[k] for k in g}
        rows += [(int(a[i]), lo + i, dz1[i]) for i in range(hi - lo)]
    ga = np.zeros((p["w1"].shape[0], items))
    for j, _, dz in sorted(rows, key=lambda t: (t[0], t[1])):
        ga[:, j] += dz
    total["w1"] = np.concatenate([total.pop("w1s"), ga], 1)
    return loss, total


@pytest.mark.parametrize("world", [1, 2, 3, 8])
@pytest.mark.parametrize("train", [False, True])
def test_row_sharded_critic_restatement_equals_the_unsharded_oracle(world, train):
    S, H, I, n = 13, 16, 50, 100
    pp, cp, tcp, batch, masks = critic_case(S, H, I, n, world + 10 * train, 1, train)
    nets = {"value_net": cp, "target_value_net": tcp, "target_policy_net": pp}
    want_loss, want, _ = CV.value_step(nets, batch, PARAMS, masks)
    loss, got = _dp_value_step(nets, batch, PARAMS, masks, world)
    assert loss == pytest.approx(want_loss, rel=1e-12)
    for k in want:
        np.testing.assert_allclose(got[k], want[k], rtol=1e-10, atol=1e-13, err_msg=k)


def _uniform(seed, draw, rows):
    """The device's draw_uniform: Philox(seed) at counter (row, (draw << 8) | 0x5a), word x >> 8, times 2^-24."""
    x = PH._philox_seeded(seed, np.asarray(rows, np.uint64), (int(draw) << 8) | 0x5A)[0]
    return (x >> np.uint32(8)).astype(np.float64) / 16777216.0


@pytest.mark.parametrize("world", [2, 3, 8])
def test_draws_at_the_row_offset_are_the_unsharded_rows(world):
    n, items, seed, draw = 130, 40, 1234567, 3
    rng = np.random.default_rng(world)
    probs = rng.dirichlet(np.ones(items), n)
    u_full = _uniform(seed, draw, np.arange(n))
    want = RO.categorical_sample(probs, u_full)[0]
    got = []
    for r in range(world):
        lo, hi = D.shard_rows(n, r, world)
        u = _uniform(seed, draw, lo + np.arange(hi - lo))
        assert np.array_equal(u, u_full[lo:hi])
        got.append(RO.categorical_sample(probs[lo:hi], u)[0])
    assert np.array_equal(np.concatenate(got), want)
