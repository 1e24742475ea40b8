"""Builders of the DiscreteActor and item-id critic cases that several GPU tests share: a DiscreteActor from numpy
parameters, the seeded item-id critic case, and that case laid out as vocabulary-shard ranks with their
DiscreteValueArgs (test_workspace_bounds_gpu.py calls the C step and phases on them to bound their workspace)."""
from __future__ import annotations

import numpy as np
import torch

import recnn_b200
from recnn_b200 import _lib
from recnn_b200.nn.arena import param_arena
from oracle import recnn_oracle as O
from oracle import reinforce_oracle as RO
from tests import _critic_vocab_oracle as CV
from tests._cuda import load_net

DEV = "cuda:0"
PARAMS = dict(gamma=0.99, min_value=-10, max_value=10)


def to_dev(x):
    return torch.from_numpy(np.ascontiguousarray(x)).to(DEV)


def make_policy(p, S, H, I):
    m = recnn_b200.nn.DiscreteActor(S, I, H)
    with torch.no_grad():
        m.linear1.weight.copy_(torch.from_numpy(p["w1"]))
        m.linear1.bias.copy_(torch.from_numpy(p["b1"]))
        m.linear2.weight.copy_(torch.from_numpy(p["w2"]))
        m.linear2.bias.copy_(torch.from_numpy(p["b2"]))
    return m.to(DEV)


class Rank:
    """One rank's nets (local dims), its SGD step and the DiscreteValueArgs of its phases."""

    def __init__(self, pp, cp, tcp, S, H, offset, num_items, rank, world, chunk, batch, masks, lr):
        L = _lib.lib()
        items = len(pp["b2"])
        self.policy = make_policy(pp, S, H, items)
        self.value = load_net(recnn_b200.nn.Critic(S, items, H), cp, DEV)
        self.target = load_net(recnn_b200.nn.Critic(S, items, H), tcp, DEV)
        self.opt = recnn_b200.optim.SGD(self.value.parameters(), lr=lr).bind(self.value)
        self.shard = _lib.VocabShard(offset, num_items, rank, world)
        self.n = n = len(batch["action"])
        self.batch, self.masks = batch, masks            # the args point into them
        a = self.args = _lib.DiscreteValueArgs()
        a.dims, a.policy_dims = _lib.Dims(S, items, H, 0), self.policy.dims
        a.learn, a.dropout = 1, int(masks is not None)
        a.chunk_items = chunk if chunk < items else items
        a.n_rows = n
        a.state, a.next_state = batch["state"].data_ptr(), batch["next_state"].data_ptr()
        a.action, a.reward, a.done = batch["action"].data_ptr(), batch["reward"].data_ptr(), batch["done"].data_ptr()
        a.value = self.opt.c_net(self.value)
        a.target_value = _lib.Net(param_arena(self.target).data_ptr(), None, None, None, None, None)
        a.target_policy = param_arena(self.policy).data_ptr()
        a.value_optim = self.opt.c_optim()
        a.gamma, a.min_value, a.max_value = PARAMS["gamma"], PARAMS["min_value"], PARAMS["max_value"]
        if masks is not None:
            a.masks[0], a.masks[1] = masks[0].data_ptr(), masks[1].data_ptr()
        self.rng_step = torch.zeros(1, dtype=torch.int64, device=DEV)
        self.losses = torch.zeros(8, device=DEV)
        a.seed, a.rng_step, a.losses = 11, self.rng_step.data_ptr(), self.losses.data_ptr()
        nbytes = L.recnn_discrete_value_workspace_bytes(a.dims, a.policy_dims, n, a.chunk_items)
        self.ws = torch.empty(nbytes, dtype=torch.uint8, device=DEV)
        a.workspace, a.workspace_bytes = self.ws.data_ptr(), nbytes

    def loss_bits(self):
        return self.losses.view(torch.int32)[[0, 4]].tolist()


def critic_case(S, H, I, n, seed, world, train):
    """(policy, critic, target critic parameters, host batch of item ids, dropout masks or None)"""
    rng = np.random.default_rng(seed)
    pp = RO.make_discrete_actor(rng, S, I, H)
    pp["w2"] = (pp["w2"] * 4).astype(np.float32)
    cp, tcp = O.make_critic(rng, S, I, H, 0.3), O.make_critic(rng, S, I, H, 0.3)
    a = rng.integers(0, I, n)
    a[:n // 4] = a[n // 4:n // 2]                                       # repeated ids
    edges = sorted({e for lo, hi in CV.item_plan(I, world) for e in (lo - 1, lo, hi - 1) if 0 <= e < I})
    a[n // 2:n // 2 + len(edges)] = edges[:n - n // 2]                  # shard edges (and chunk edges inside them)
    batch = {"state": rng.normal(0, 1, (n, S)).astype(np.float32), "next_state": rng.normal(0, 1, (n, S)).astype(np.float32),
             "action": a, "reward": (rng.integers(1, 6, n) - 3).astype(np.float32),
             "done": (rng.random(n) < 0.1).astype(np.float32)}
    masks = [(rng.random((n, H)) >= 0.5).astype(np.uint8) for _ in range(2)] if train else None
    return pp, cp, tcp, batch, masks


def critic_ranks(pp, cp, tcp, S, H, I, world, chunk, batch, masks, lr=1e-2):
    """(the W ranks of a critic_case, the device batch, the device masks)"""
    dev_batch = {k: to_dev(v) for k, v in batch.items()}
    dev_masks = None if masks is None else [to_dev(m) for m in masks]
    return [Rank(ps, c, tc, S, H, ps["offset"], I, r, world, chunk, dev_batch, dev_masks, lr)
            for r, (ps, c, tc) in enumerate(zip(RO.shard_policy(pp, world), CV.shard_critic(cp, S, world),
                                                CV.shard_critic(tcp, S, world)))], dev_batch, dev_masks
