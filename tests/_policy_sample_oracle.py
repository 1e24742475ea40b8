"""float64 restatement of the REINFORCE policy's sampled slates (DiscreteActor.sample_topk /
recnn_discrete_sample_topk) and of their vocabulary-sharded form (recnn_discrete_shard_sample_topk +
recnn_discrete_shard_sample_topk_finish).

A slate is the top-k of the perturbed logits z + G (Gumbel-top-k): G = -log(-log u) of item i in global row r, with u
from the same Philox bits as the device (tests/_philox.py) at counter (i, r << 8 | 0x67), u = (2 m + 1) 2^-24 with m
the top 23 bits of output word x; the logs are taken in float64.  Selection and exclusion are _policy_topk_oracle's on
z + G (larger first, equal keys to the smaller id); values are pi = exp(z - M) / S of the returned ids over every
item; missing slots are id -1, value 0."""
from __future__ import annotations

import numpy as np

from tests import _philox as PX
from tests import _policy_topk_oracle as TK

TAG = 0x67
G_MAX = 16.75          # csrc/reinforce.cuh kGumbelMax: no fp32 G exceeds it


def uniforms(seed, rows, n_items):
    """float64 [len(rows), n_items]: the u of items 0..n_items-1 in the given global rows."""
    rows = np.asarray(rows, dtype=np.uint64).reshape(-1, 1)
    ids = np.arange(n_items, dtype=np.uint64).reshape(1, -1)
    hi = (rows << np.uint64(8)) | np.uint64(TAG)
    seed = int(seed) & 0xFFFFFFFFFFFFFFFF
    x = PX.philox4x32_10((ids, np.uint64(0), hi & np.uint64(0xFFFFFFFF), hi >> np.uint64(32)),
                         (seed & 0xFFFFFFFF, seed >> 32))[0]
    x = np.broadcast_to(x, (rows.shape[0], n_items))
    return (2.0 * (x >> np.uint32(9)).astype(np.float64) + 1.0) * 2.0 ** -24


def gumbel(seed, rows, n_items):
    return -np.log(-np.log(uniforms(seed, rows, n_items)))


def perturbed(z, seed, row0=0):
    """z + G of every item of z's rows, whose global rows are row0 .. row0 + N - 1 (row0 an int) or row0 (an array)."""
    rows = np.arange(row0, row0 + z.shape[0]) if np.isscalar(row0) else np.asarray(row0)
    return z + gumbel(seed, rows, z.shape[1])


def _values(z, ids):
    M = z.max(1, keepdims=True)
    S = np.exp(z - M).sum(1, keepdims=True)
    v = np.exp(np.take_along_axis(z, np.maximum(ids, 0), 1) - M) / S
    return np.where(ids >= 0, v, 0.0)


def sample_topk(z, k, seed, exclude=None, row0=0):
    """(values float64 [N, k], ids int64 [N, k], perturbed keys [N, k]) of the unsharded call on float64 logits z."""
    g = perturbed(z, seed, row0)
    top_g, top_i = TK._select(g, k, TK._eligible(z, exclude))
    return _values(z, top_i), top_i, top_g


def shard_sample_topk(z, k, world, seed, exclude=None, row0=0):
    """The sharded restatement: per rank the best k of its block by z + G with global ids (padded with (-inf, -1)),
    then a k-way merge of the W lists; values from the logits of the winners."""
    g = perturbed(z, seed, row0)
    cand_g, cand_i = [], []
    for lo, hi in TK.item_plan(z.shape[1], world):
        tg, ti = TK._select(g[:, lo:hi], k, TK._eligible(z[:, lo:hi], exclude, lo), lo)
        cand_g.append(tg)
        cand_i.append(ti)
    cand_g, cand_i = np.concatenate(cand_g, 1), np.concatenate(cand_i, 1)
    n = z.shape[0]
    top_i = np.full((n, k), -1, dtype=np.int64)
    for r in range(n):
        live = cand_i[r] >= 0
        gi, ii = cand_g[r, live], cand_i[r, live]
        order = np.lexsort((ii, -gi))[:k]
        top_i[r, :len(order)] = ii[order]
    return _values(z, top_i), top_i


def determined(top_g, k, bar):
    """([N, k] bool, [N] bool) from the sorted perturbed keys of a row's best k + 1 (or all) eligible items: slot j is
    settled in fp32 when its key is more than `bar` from both neighbours (so no error of `bar` can move its item), and
    the slate's id set when the k-th / (k+1)-th gap exceeds `bar`."""
    with np.errstate(invalid="ignore"):
        d = top_g[:, :-1] - top_g[:, 1:]
    d = np.where(np.isfinite(d), d, np.inf)
    n = top_g.shape[0]
    below = np.concatenate([d, np.full((n, k + 1 - top_g.shape[1]), np.inf)], 1)[:, :k]
    above = np.concatenate([np.full((n, 1), np.inf), below[:, :k - 1]], 1)
    return (above > bar) & (below > bar), below[:, k - 1] > bar


def plackett_luce(p, draws):
    """{ordered tuple of the first `draws` ids: probability} of drawing without replacement from weights p (brute
    force over every ordered tuple; p's zero entries are never drawn)."""
    out = {}

    def walk(prefix, mass, left):
        if len(prefix) == draws:
            out[tuple(prefix)] = mass
            return
        tot = sum(p[j] for j in left)
        for j in left:
            if p[j] > 0:
                walk(prefix + [j], mass * p[j] / tot, [x for x in left if x != j])
    walk([], 1.0, list(range(len(p))))
    return out
