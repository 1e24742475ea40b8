"""float64 oracle of the vocabulary-parallel REINFORCE policy as the device computes it (recnn_reinforce_shard_* and
recnn_discrete_shard_* in include/recnn_b200.h), built on oracle/reinforce_oracle.py.

oracle.reinforce_oracle.sharded_policy_grad all-reduces dh [rows, H] (exchange 2).  The device instead has every rank
back-propagate its own dh_r = (dz_r W2_r) * [h > 0] into its own layer-1 gradient dW1_r = dh_r^T x, db1_r, and
all-reduces that block: the ReLU gate is the same on every rank, so the sum is linear and the result is the same, while
the message is H * (pad4(S) + 1) floats whatever the number of rows.  The sharded draw picks the rank whose share of
the cumulative mass holds u, then draws inside that rank's block at the conditional uniform."""
from __future__ import annotations

import numpy as np

from oracle import reinforce_oracle as RO


def shard_stats(shards, state, action):
    """Per rank: hidden h, logits z and the record (m, s, za) of exchange 1."""
    x = state.astype(np.float64)
    n = state.shape[0]
    out = []
    for sh in shards:
        h = np.maximum(x @ sh["w1"].astype(np.float64).T + sh["b1"].astype(np.float64), 0)
        z = h @ sh["w2"].astype(np.float64).T + sh["b2"].astype(np.float64)
        cnt = z.shape[1]
        m = z.max(axis=1)
        s = np.exp(z - m[:, None]).sum(axis=1)
        mine = (action >= sh["offset"]) & (action < sh["offset"] + cnt)
        za = np.where(mine, z[np.arange(n), np.clip(action - sh["offset"], 0, cnt - 1)], 0.0)
        out.append({"h": h, "z": z, "m": m, "s": s, "za": za, "mine": mine})
    return out


def merge(local):
    """Rank-order merge of the gathered records: M = max m_q, S = sum s_q exp(m_q - M), za = sum za_q."""
    M = np.max([r["m"] for r in local], axis=0)
    S = np.sum([r["s"] * np.exp(r["m"] - M) for r in local], axis=0)
    za = np.sum([r["za"] for r in local], axis=0)
    return M, S, za


def sharded_policy_grad_layer1(shards, state, action, beta_logp, ret, method, K=10):
    """Loss and per-rank gradients with exchange 2 as the all-reduce of the ranks' layer-1 gradients."""
    x = state.astype(np.float64)
    local = shard_stats(shards, state, action)
    M, S, za = merge(local)
    L, g, _ = RO.row_terms(np.exp(za - M) / S, beta_logp, ret, method, K)
    grads = []
    for sh, r in zip(shards, local):
        dz = -np.exp(r["z"] - M[:, None]) / S[:, None] * g[:, None]
        rows = np.nonzero(r["mine"])[0]
        dz[rows, action[rows] - sh["offset"]] += g[rows]
        dh = (dz @ sh["w2"].astype(np.float64)) * (r["h"] > 0)
        grads.append({"w2": dz.T @ r["h"], "b2": dz.sum(0), "w1_r": dh.T @ x, "b1_r": dh.sum(0)})
    w1, b1 = grads[0]["w1_r"].copy(), grads[0]["b1_r"].copy()       # the all-reduce, in rank order
    for gr in grads[1:]:
        w1 += gr["w1_r"]
        b1 += gr["b1_r"]
    for gr in grads:
        gr["w1"], gr["b1"] = w1, b1
    return float(L.sum()), grads


def sharded_sample(blocks, offsets, uniforms):
    """The sharded inverse-CDF draw.  blocks: every rank's column block [n, cnt_q] of the (globally normalised)
    probabilities; returns the global ids."""
    n = blocks[0].shape[0]
    mass = np.stack([b.astype(np.float64).sum(axis=1) for b in blocks], axis=1)      # [n, W]
    ids = np.empty(n, np.int64)
    for r in range(n):
        u = float(uniforms[r])
        c = np.cumsum(mass[r])
        live = np.nonzero(mass[r] > 0)[0]
        over = [q for q in live if c[q] > u]
        q = over[0] if over else live[-1]
        before = c[q] - mass[r, q]
        u2 = min((u - before) / mass[r, q], np.nextafter(1.0, 0.0))
        a, _, _ = RO.categorical_sample(blocks[q][r:r + 1], np.array([u2]))
        ids[r] = offsets[q] + int(a[0])
    return ids
