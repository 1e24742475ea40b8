"""Float64 restatement of one Beta call sharded over the item vocabulary (recnn_beta_shard_* in include/recnn_b200.h):
begin (local logits, max, sum and the target's logit) -> all-gather -> rows (rank-order merge, the block of p, its
partial sums of expm1(p) and p expm1(p)) -> all-gather -> end (T, U, p_a, loss, the block's dW / db).  Each rank sees
only its rows of the weight and the gathered records, so this checks that the two exchanges carry everything the
unsharded call (oracle/beta_oracle.loss_and_grads) needs."""
from __future__ import annotations

import numpy as np


def item_plan(items, world):
    """[lo, hi) of every rank: blocks of ceil(items / world), the last one shorter (recnn_b200.dist.vocab_shard)."""
    per = -(-items // world)
    return [(min(r * per, items), min((r + 1) * per, items)) for r in range(world)]


def sharded_call(w, b, state, ids, world, order=None):
    """Every rank's (block of p [N, hi - lo], loss, dW block, db block, error bits).  ``order``: the rank order the
    gathered records arrive in (a wrong order sets bit 2)."""
    s = np.asarray(state, np.float64)
    ids = np.asarray(ids, np.int64)
    n, items = s.shape[0], w.shape[0]
    rows = np.arange(n)
    plan = item_plan(items, world)
    order = list(range(world)) if order is None else order
    # begin: the local logits and the exchange-1 record {lo, hi, items, n; m, s, z_a}
    z, rec1 = [], []
    for lo, hi in plan:
        zr = s @ np.asarray(w[lo:hi], np.float64).T + np.asarray(b[lo:hi], np.float64)
        m = zr.max(1)
        mine = (ids >= lo) & (ids < hi)
        za = np.zeros(n)
        za[mine] = zr[rows[mine], ids[mine] - lo]
        z.append(zr)
        rec1.append(((lo, hi, items, n), m, np.exp(zr - m[:, None]).sum(1), za))
    g1 = [rec1[q] for q in order]

    def plan_bad(g, r):
        expect, bad = 0, False
        for q, (h, *_) in enumerate(g):
            bad = bad or h[0] != expect or h[1] <= h[0] or h[2] != items or h[3] != n
            expect = h[1]
            if q == r:
                bad = bad or h[:2] != plan[r]
        return bad or expect != items

    # rows: the rank-order merge, the block of p, the exchange-2 record {header; s1, s2, 0}
    M = np.max([g[1] for g in g1], 0)
    S = sum(g[2] * np.exp(g[1] - M) for g in g1)
    ZA = sum(g[3] for g in g1)
    p, rec2 = [], []
    for r, (lo, hi) in enumerate(plan):
        pr = np.exp(z[r] - M[:, None]) / S[:, None]
        em = np.expm1(pr)
        p.append(pr)
        rec2.append(((lo, hi, items, n), em.sum(1), (pr * em).sum(1)))
    g2 = [rec2[q] for q in order]
    # end
    T = items + sum(g[1] for g in g2)
    U = sum(g[2] for g in g2)
    ok = (ids >= 0) & (ids < items)
    pa = np.where(ok, np.exp(ZA - M) / S, 0.0)
    loss = float(np.mean(np.where(ok, np.log(T) - pa, 0.0)))
    out = []
    for r, (lo, hi) in enumerate(plan):
        pr = p[r]
        dz = pr / n * ((np.expm1(pr) - U[:, None]) / T[:, None] + pa[:, None])
        mine = ok & (ids >= lo) & (ids < hi)
        dz[rows[mine], ids[mine] - lo] -= pr[rows[mine], ids[mine] - lo] / n
        dz[~ok] = 0.0
        err = (0 if ok.all() else 1) | (2 if plan_bad(g1, r) or plan_bad(g2, r) else 0)
        out.append((pr, loss, dz.T @ s, dz.sum(0), err))
    return out
