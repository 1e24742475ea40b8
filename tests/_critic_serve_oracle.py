"""Float64 restatement of serving through the DDPG / TD3 critic (``Critic.topk`` / ``Critic.rank``).

Q of a pair is ``oracle.recnn_oracle.critic_forward`` in eval mode (no dropout masks).  ``q_pairs`` evaluates it in the
split form the kernels use (a per-row and a per-item term of layer 1) so that thousands of pairs per row stay cheap;
``q_pairs_direct`` is the plain forward on [state | action] rows, and the host tests check the two agree.

The rules: a row's columns are its candidates (-1: padding) or every item; excluded ids are never returned; the order
is higher Q first, equal Q the smaller id first; a row with fewer than k eligible columns ends in id -1, value
-FLT_MAX.  ``rank`` counts the eligible columns that beat the target; the target is never excluded, and a target
missing from its row's candidates gets the row's count of eligible candidates.
"""
from __future__ import annotations

import numpy as np

from oracle.recnn_oracle import critic_forward

FLT_MAX = float(np.finfo(np.float32).max)


def params64(critic):
    """The critic's weights as the float64 dict critic_forward takes."""
    g = lambda t: t.detach().cpu().double().numpy()
    return {"w1": g(critic.linear1.weight), "b1": g(critic.linear1.bias), "w2": g(critic.linear2.weight),
            "b2": g(critic.linear2.bias), "w3": g(critic.linear3.weight), "b3": g(critic.linear3.bias)}


def all_ids(n, n_items):
    return np.broadcast_to(np.arange(n_items, dtype=np.int64), (n, n_items))


def q_pairs_direct(p, state, table, ids):
    """float64 [N, M]: critic_forward(state[r], table[ids[r, j]]) (nan for padding), one row at a time."""
    state, table, ids = np.asarray(state, np.float64), np.asarray(table, np.float64), np.asarray(ids)
    out = np.full(ids.shape, np.nan)
    for r in range(ids.shape[0]):
        ok = ids[r] >= 0
        if ok.any():
            q, _ = critic_forward(p, np.repeat(state[r:r + 1], int(ok.sum()), 0), table[ids[r][ok]])
            out[r, ok] = q[:, 0]
    return out


def q_pairs(p, state, table, ids, rows_per_step=16):
    """q_pairs_direct through the split of layer 1: u = W1[:, :S] s + b1, v = W1[:, S:] e, h1 = relu(u + v)."""
    state, table, ids = np.asarray(state, np.float64), np.asarray(table, np.float64), np.asarray(ids)
    S = state.shape[1]
    u = state @ p["w1"][:, :S].T + p["b1"]
    out = np.full(ids.shape, np.nan)
    for r0 in range(0, ids.shape[0], rows_per_step):
        blk = ids[r0:r0 + rows_per_step]
        v = table[np.where(blk >= 0, blk, 0)] @ p["w1"][:, S:].T               # [nr, M, H]
        h1 = np.maximum(u[r0:r0 + rows_per_step, None, :] + v, 0.0)
        h2 = np.maximum(h1 @ p["w2"].T + p["b2"], 0.0)
        q = (h2 @ p["w3"].T)[..., 0] + p["b3"][0]
        out[r0:r0 + rows_per_step] = np.where(blk >= 0, q, np.nan)
    return out


def _eligible(ids_row, q_row, ex_row):
    ex = set() if ex_row is None else set(int(x) for x in ex_row)
    return [(float(q), int(i)) for q, i in zip(q_row, ids_row) if i >= 0 and int(i) not in ex]


def order(q_row, ids_row, ex_row=None):
    """The eligible (q, id) of one row, best first: higher q, then the smaller id."""
    el = _eligible(ids_row, q_row, ex_row)
    return sorted(el, key=lambda t: (-t[0], t[1]))


def topk(q, ids, k, exclude=None):
    """(values float64 [N, k], ids int64 [N, k]) by the rules above; exclude: one id list per row (or None)."""
    n = q.shape[0]
    vals = np.full((n, k), -FLT_MAX)
    out = np.full((n, k), -1, np.int64)
    for r in range(n):
        best = order(q[r], ids[r], None if exclude is None else exclude[r])[:k]
        for j, (v, i) in enumerate(best):
            vals[r, j], out[r, j] = v, i
    return vals, out


def rank(q, ids, target, exclude=None):
    """int64 [N]: the eligible columns that beat target[r]; the target itself is never excluded.  q / ids must hold
    the target's column when it is among the row's candidates (all items: always)."""
    n = q.shape[0]
    out = np.zeros(n, np.int64)
    for r in range(n):
        t = int(target[r])
        ex = set() if exclude is None else set(int(x) for x in exclude[r]) - {t}
        el = _eligible(ids[r], q[r], sorted(ex))
        hit = [v for v, i in el if i == t]
        if not hit:
            out[r] = len(el)
            continue
        qt = hit[0]
        out[r] = sum(1 for v, i in el if i != t and (v > qt or (v == qt and i < t)))
    return out
