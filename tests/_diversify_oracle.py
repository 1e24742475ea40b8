"""float64 restatement of diversified re-ranking (recnn_slate_diversify, recnn_b200.utils.diversify).

``Greedy`` holds one pool row's greedy state; ``objective()`` gives every column's objective after the picks so far
(NaN where a column is not eligible), ``pick(col)`` applies a pick.  ``greedy`` runs it to k picks with the kernel's
tie rule (larger objective, then smaller id, then smaller column) and the DPP's stopping rule.  The GPU tests replay
the kernel's own picks through ``Greedy`` to certify each one against the float64 objective."""
from __future__ import annotations

import numpy as np

DPP_EPS = 1e-4


def cosine_sim(X):
    """[m, m] cosine similarity of the rows of X, clipped to [-1, 1], 0 wherever a zero vector is involved."""
    X = np.asarray(X, dtype=np.float64)
    n = np.sqrt((X * X).sum(1))
    den = np.outer(n, n)
    sim = np.where(den > 0, (X @ X.T) / np.where(den > 0, den, 1.0), 0.0)
    return np.clip(sim, -1.0, 1.0)


class Greedy:
    def __init__(self, ids, scores, table, method, weight):
        self.ids = np.asarray(ids, dtype=np.int64)
        self.s = np.asarray(scores, dtype=np.float64)
        m = self.ids.shape[0]
        X = np.zeros((m, np.asarray(table).shape[1]))
        ok = self.ids >= 0
        X[ok] = np.asarray(table, dtype=np.float64)[self.ids[ok]]
        self.sim = cosine_sim(X)
        self.S = 0.5 * (1.0 + self.sim)
        self.w = float(weight)
        self.dpp = method == "dpp" and self.w < 1.0
        self.alive = ok.copy()
        self.t = 0
        self.ms = np.full(m, -np.inf)                 # MMR: max similarity to the picks
        self.d2 = np.diag(self.S).copy()              # DPP: Schur complement of each column in S
        self.c = np.zeros((m, 0))                     # DPP: the incremental Cholesky rows

    def objective(self):
        with np.errstate(divide="ignore", invalid="ignore"):
            if self.dpp:
                obj = self.w / (1.0 - self.w) * self.s + np.where(self.d2 > 0, np.log(np.maximum(self.d2, 1e-300)),
                                                                   -np.inf)
            elif self.t == 0:
                obj = self.w * self.s
            else:
                obj = self.w * self.s - (1.0 - self.w) * self.ms
        return np.where(self.alive, obj, np.nan)

    def best(self, obj=None):
        """The column the tie rule picks, or None when nothing is eligible."""
        obj = self.objective() if obj is None else obj
        cols = np.nonzero(self.alive)[0]
        if cols.size == 0:
            return None
        order = np.lexsort((cols, self.ids[cols], -obj[cols]))
        return int(cols[order[0]])

    def pick(self, col):
        j = int(col)
        if self.dpp:
            e = (self.S[:, j] - self.c @ self.c[j]) / np.sqrt(self.d2[j])
            self.c = np.concatenate([self.c, e[:, None]], axis=1)
            self.d2 = self.d2 - e * e
        else:
            self.ms = np.maximum(self.ms, self.sim[:, j])
        self.alive &= self.ids != self.ids[j]
        self.t += 1


def greedy(ids, scores, table, k, method, weight):
    """(ids [k], pos [k], gain [k]) of one pool row in float64; -1 / -1 / NaN past the end."""
    g = Greedy(ids, scores, table, method, weight)
    out_ids, out_pos, gain = np.full(k, -1), np.full(k, -1), np.full(k, np.nan)
    for t in range(k):
        obj = g.objective()
        j = g.best(obj)
        if j is None or (g.dpp and g.d2[j] < DPP_EPS):
            break
        out_ids[t], out_pos[t], gain[t] = g.ids[j], j, obj[j]
        g.pick(j)
    return out_ids, out_pos, gain


def greedy_rows(ids, scores, table, k, method, weight):
    """greedy over every row of [N, m] pools: (ids, pos, gain), each [N, k]."""
    rows = [greedy(i, s, table, k, method, weight) for i, s in zip(ids, scores)]
    return tuple(np.stack(x) for x in zip(*rows))
