"""float64 restatement of the REINFORCE policy's top-k (DiscreteActor.topk / recnn_discrete_topk) and of its
vocabulary-sharded form (recnn_discrete_shard_topk + recnn_discrete_shard_topk_finish).

Ranking: logit descending, equal logits to the smaller id; excluded ids (negative ones are padding) are never returned
but stay in the normaliser; values pi = exp(z - M) / S over every item; missing slots are id -1, value 0."""
from __future__ import annotations

import numpy as np

from oracle import reinforce_oracle as RO


def logits(p, state):
    """[N, num_items] float64 logits of the policy with parameters p."""
    _, h = RO.discrete_forward(p, state)
    return h @ p["w2"].astype(np.float64).T + p["b2"].astype(np.float64)


def _eligible(z, exclude, id0=0):
    """[N, w] bool: item id0 + j of row r is not excluded."""
    ok = np.ones(z.shape, dtype=bool)
    if exclude is not None:
        for r, row in enumerate(np.asarray(exclude)):
            local = row[(row >= id0) & (row < id0 + z.shape[1])] - id0
            ok[r, local] = False
    return ok


def _select(z, k, ok, id0=0):
    """(logits [N, k], ids [N, k]) of the best k eligible items per row by a stable argsort of -z; missing slots are
    (-inf, -1)."""
    n = z.shape[0]
    top_z = np.full((n, k), -np.inf)
    top_i = np.full((n, k), -1, dtype=np.int64)
    for r in range(n):
        order = np.argsort(-z[r], kind="stable")
        order = order[ok[r, order]][:k]
        top_z[r, :len(order)] = z[r, order]
        top_i[r, :len(order)] = order + id0
    return top_z, top_i


def _values(top_z, top_i, M, S):
    v = np.exp(top_z - M[:, None]) / S[:, None]
    return np.where(top_i >= 0, v, 0.0)


def topk(z, k, exclude=None):
    """(values float64 [N, k], ids int64 [N, k]) of the unsharded call on float64 logits z [N, num_items]."""
    M = z.max(1)
    S = np.exp(z - M[:, None]).sum(1)
    top_z, top_i = _select(z, k, _eligible(z, exclude))
    return _values(top_z, top_i, M, S), top_i


def item_plan(num_items, world):
    """recnn_b200.dist.vocab_shard's blocks: ceil(num_items / world) items each, the last one shorter."""
    per = -(-num_items // world)
    return [(min(q * per, num_items), min((q + 1) * per, num_items)) for q in range(world)]


def shard_topk(z, k, world, exclude=None):
    """The sharded restatement: per rank, the local (max, sum of exp) and the local best k with global ids (padded with
    (-inf, -1) when its block holds fewer); then M, S merged in rank order and a k-way merge of the W lists."""
    recs = []
    for lo, hi in item_plan(z.shape[1], world):
        zl = z[:, lo:hi]
        m = zl.max(1)
        s = np.exp(zl - m[:, None]).sum(1)
        recs.append((m, s) + _select(zl, k, _eligible(zl, exclude, lo), lo))
    M = np.max([r[0] for r in recs], 0)
    S = sum(r[1] * np.exp(r[0] - M) for r in recs)
    cand_z = np.concatenate([r[2] for r in recs], 1)
    cand_i = np.concatenate([r[3] for r in recs], 1)
    n = z.shape[0]
    top_z = np.full((n, k), -np.inf)
    top_i = np.full((n, k), -1, dtype=np.int64)
    for r in range(n):
        live = cand_i[r] >= 0
        zi, ii = cand_z[r, live], cand_i[r, live]
        order = np.lexsort((ii, -zi))[:k]
        top_z[r, :len(order)] = zi[order]
        top_i[r, :len(order)] = ii[order]
    return _values(top_z, top_i, M, S), top_i


def boundary_gap(z, k, exclude=None):
    """[N]: the gap between the k-th and (k+1)-th eligible logit of every row (inf when fewer than k + 1 are
    eligible): the ids of a row are only determined in fp32 when this exceeds the fp32 error of the logits."""
    top_z, _ = _select(z, min(k + 1, z.shape[1]), _eligible(z, exclude))
    if k + 1 > z.shape[1]:
        return np.full(z.shape[0], np.inf)
    gap = top_z[:, k - 1] - top_z[:, k]
    return np.where(np.isfinite(top_z[:, k]), gap, np.inf)
