"""float64 oracle of the item-id REINFORCE critic step sharded over the item vocabulary, as the device computes it
(recnn_discrete_value_shard_* in include/recnn_b200.h), and of the unsharded one-hot step it must equal.

Rank r of W holds items [lo_r, hi_r) = vocab_shard(num_items, r, W): rows [lo_r, hi_r) of the target policy's linear2
and columns S + [lo_r, hi_r) of both critics' linear1 (a Critic(S, hi_r - lo_r, H)); everything else is replicated.
Layer 1's pre-activation is a state-block product plus an [N, H] action term, a sum over items, hence over ranks:
  * online term  add_r[m] = W1a[:, a_m - lo_r] when rank r holds a_m, else 0 (exactly one rank contributes per row);
  * target term  Y_r = sum_local exp(z - m_r) W1a'^T with the rank's (m_r, s_r); after the all-gather of (m, s):
                 M = max m_q, S = sum_q s_q exp(m_q - M) in rank order, Y_r <- Y_r exp(m_r - M) / S;
  * one all-reduce of {Y_r, add_r}: from there to dz1 every rank computes the same thing, so the replicated gradients
    need no exchange, and the action block's gradient is the rank's own columns of dz1^T one-hot(a)."""
from __future__ import annotations

import numpy as np

from oracle import reinforce_oracle as RO

F64 = np.float64
RO_KEYS = ("w1", "b1", "w2", "b2", "w3", "b3")


def item_plan(num_items, world):
    """[(lo, hi)] of every rank: recnn_b200.dist.vocab_shard's plan, through the oracle's split of the policy."""
    split = RO.shard_policy({"w1": 0, "b1": 0, "w2": np.zeros((num_items, 1)), "b2": np.zeros(num_items)}, world)
    return [(sh["offset"], sh["offset"] + len(sh["b2"])) for sh in split]


def shard_critic(p, S, world):
    """The critic's per-rank arenas: linear1 = [W1s | W1a[:, lo:hi]], the rest replicated; "offset" = lo."""
    items = p["w1"].shape[1] - S
    out = []
    for lo, hi in item_plan(items, world):
        q = dict(p)
        q["w1"] = np.concatenate([p["w1"][:, :S], p["w1"][:, S + lo:S + hi]], 1)
        q["offset"] = lo
        out.append(q)
    return out


def _hidden(z, mask):
    h = np.maximum(z, 0.0)
    return h if mask is None else h * (np.asarray(mask, F64) * 2.0)


def _critic_tail(p, S, x, term, masks):
    """q [N, 1] and the cache of the critic with layer 1's action block given as its [N, H] term."""
    m1, m2 = masks if masks is not None else (None, None)
    w = {k: np.asarray(p[k], F64) for k in RO_KEYS}
    h1 = _hidden(x @ w["w1"][:, :S].T + term + w["b1"], m1)
    h2 = _hidden(h1 @ w["w2"].T + w["b2"], m2)
    return h2 @ w["w3"].T + w["b3"], (h1, h2, m1, m2, w)


def _backward(S, x, cache, dq):
    """Gradients of the replicated blocks and dz1 [N, H] (the action block is the caller's)."""
    h1, h2, m1, m2, w = cache
    g = {"w3": dq.T @ h2, "b3": dq.sum(0)}
    dz2 = (dq @ w["w3"]) * (h2 > 0) * (2.0 if m2 is not None else 1.0)
    g["w2"], g["b2"] = dz2.T @ h1, dz2.sum(0)
    dz1 = (dz2 @ w["w2"]) * (h1 > 0) * (2.0 if m1 is not None else 1.0)
    g["w1s"], g["b1"] = dz1.T @ x, dz1.sum(0)
    return g, dz1


def _td(batch, q2, params):
    r, d = (np.asarray(batch[k], F64).reshape(-1, 1) for k in ("reward", "done"))
    y = r + (1.0 - d) * params["gamma"] * q2
    return np.clip(y, params["min_value"], params["max_value"])


def value_step(nets, batch, params, masks=None):
    """The unsharded critic step with the dense one-hot action, float64: (loss, gradients of value_net, oob)."""
    p, tp, tv = nets["value_net"], nets["target_policy_net"], nets["target_value_net"]
    S = tp["w1"].shape[1]
    x, x2 = (np.asarray(batch[k], F64) for k in ("state", "next_state"))
    a = np.asarray(batch["action"])
    n, items = len(a), tp["w2"].shape[0]
    ok = (a >= 0) & (a < items)
    onehot = np.zeros((n, items))
    onehot[np.nonzero(ok)[0], a[ok]] = 1.0
    probs, _ = RO.discrete_forward(tp, x2)
    q2, _ = _critic_tail(tv, S, x2, probs @ np.asarray(tv["w1"], F64)[:, S:].T, None)
    y = _td(batch, q2, params)
    q, cache = _critic_tail(p, S, x, onehot @ np.asarray(p["w1"], F64)[:, S:].T, masks)
    diff = q - y
    g, dz1 = _backward(S, x, cache, 2.0 * diff / n)
    g["w1"] = np.concatenate([g.pop("w1s"), dz1.T @ onehot], 1)
    return float(np.mean(diff * diff)), g, bool((~ok).any())


def sharded_value_step(cshards, tcshards, pshards, batch, params, masks=None):
    """The same step on W ranks, phase by phase (begin / all-gather / merge / all-reduce / end).  Returns (losses,
    per-rank gradients (linear1 with the local action block), oob flags, the all-reduced terms {Y, add})."""
    S = pshards[0]["w1"].shape[1]
    x, x2 = (np.asarray(batch[k], F64) for k in ("state", "next_state"))
    a = np.asarray(batch["action"])
    n = len(a)
    num_items = sum(len(sh["b2"]) for sh in pshards)
    begin = []
    for ps, tc, c in zip(pshards, tcshards, cshards):                         # ---- begin (rank-local)
        lo, cnt = ps["offset"], len(ps["b2"])
        h = np.maximum(x2 @ np.asarray(ps["w1"], F64).T + np.asarray(ps["b1"], F64), 0)
        z = h @ np.asarray(ps["w2"], F64).T + np.asarray(ps["b2"], F64)
        m = z.max(axis=1)
        e = np.exp(z - m[:, None])
        Y = e @ np.asarray(tc["w1"], F64)[:, S:].T                          # unnormalised
        mine = (a >= lo) & (a < lo + cnt)
        add = np.zeros((n, c["w1"].shape[0]))
        add[mine] = np.asarray(c["w1"], F64)[:, S + a[mine] - lo].T
        begin.append({"m": m, "s": e.sum(axis=1), "Y": Y, "add": add, "mine": mine, "lo": lo})
    M = np.max([b["m"] for b in begin], axis=0)                               # ---- all-gather + merge, rank order
    Ssum = np.zeros(n)
    for b in begin:
        Ssum = Ssum + b["s"] * np.exp(b["m"] - M)
    Y = np.zeros_like(begin[0]["Y"])                                          # ---- all-reduce, rank order
    add = np.zeros_like(Y)
    for b in begin:
        Y = Y + b["Y"] * np.exp(b["m"] - M)[:, None] / Ssum[:, None]
        add = add + b["add"]
    oob = bool(((a < 0) | (a >= num_items)).any())
    losses, grads = [], []
    for b, tc, c in zip(begin, tcshards, cshards):                            # ---- end (replicated but the scatter)
        q2, _ = _critic_tail(tc, S, x2, Y, None)
        y = _td(batch, q2, params)
        q, cache = _critic_tail(c, S, x, add, masks)
        diff = q - y
        g, dz1 = _backward(S, x, cache, 2.0 * diff / n)
        block = np.zeros((dz1.shape[1], c["w1"].shape[1] - S))
        for row in np.nonzero(b["mine"])[0]:                                  # ascending rows per column
            block[:, a[row] - b["lo"]] += dz1[row]
        g["w1"] = np.concatenate([g.pop("w1s"), block], 1)
        losses.append(float(np.mean(diff * diff)))
        grads.append(g)
    return losses, grads, [oob] * len(begin), {"Y": Y, "add": add}
