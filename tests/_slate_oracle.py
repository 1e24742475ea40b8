"""Float64 restatement of the slate evaluation (recnn_slate_distances in include/recnn_b200.h, slate_metrics in
recnn_b200/utils/metrics.py): the pairwise distance matrix of each slate, its per-row reductions, and the exposure,
coverage and novelty metrics, in plain numpy."""
from __future__ import annotations

import numpy as np


def distance_matrices(ids, table, metric):
    """float64 [N, k, k]: scipy's cdist metric between the slots' table rows, except that a cosine pair with a zero
    vector is 1 (scipy: NaN); 0 on the diagonal of filled slots, NaN wherever an empty slot (-1) is involved."""
    ids = np.asarray(ids, dtype=np.int64)
    t = np.asarray(table, dtype=np.float64)
    n, k = ids.shape
    x = t[np.where(ids >= 0, ids, 0)]                                   # [N, k, D]
    if metric == "euclidean":
        diff = x[:, :, None, :] - x[:, None, :, :]
        m = np.sqrt((diff * diff).sum(-1))
    else:
        nrm = np.sqrt((x * x).sum(-1))
        dot = np.einsum("nid,njd->nij", x, x)
        den = nrm[:, :, None] * nrm[:, None, :]
        with np.errstate(divide="ignore", invalid="ignore"):
            m = np.clip(1.0 - dot / den, 0.0, 2.0)
        m = np.where(den == 0, 1.0, m)
    filled = ids >= 0
    both = filled[:, :, None] & filled[:, None, :]
    m = np.where(both, m, np.nan)
    eye = np.eye(k, dtype=bool)[None]
    return np.where(eye & both, 0.0, m)


def row_stats(ids, matrices):
    """(mean, min, count) per row over the unordered pairs i < j of filled slots; NaN below two filled slots."""
    ids = np.asarray(ids)
    n, k = ids.shape
    count = (ids >= 0).sum(1)
    iu = np.triu_indices(k, 1)
    mean = np.full(n, np.nan)
    mn = np.full(n, np.nan)
    for r in range(n):
        if count[r] >= 2:
            v = matrices[r][iu]
            v = v[~np.isnan(v)]
            mean[r], mn[r] = v.mean(), v.min()
    return mean, mn, count


def slate_metrics(ids, n_items, table=None, metric="cosine", popularity=None, n_users=None):
    """The dict of recnn_b200.utils.metrics.slate_metrics, in float64."""
    ids = np.asarray(ids, dtype=np.int64)
    filled = ids[ids >= 0]
    c = np.bincount(filled, minlength=n_items).astype(np.float64)
    out = {"coverage": float((c > 0).sum()) / n_items, "rows": int(ids.shape[0]), "slots": int(filled.size)}
    total = c.sum()
    if total > 0:
        cs = np.sort(c)
        i = np.arange(1, n_items + 1, dtype=np.float64)
        out["gini"] = float(((2 * i - n_items - 1) * cs).sum() / (n_items * total))
        p = c[c > 0] / total
        out["exposure_entropy"] = float(-(p * np.log2(p)).sum())
    else:
        out["gini"] = out["exposure_entropy"] = float("nan")
    if table is not None:
        mean, mn, count = row_stats(ids, distance_matrices(ids, table, metric))
        ok = count >= 2
        out["ild"] = float(mean[ok].mean()) if ok.any() else float("nan")
        out["ild_min"] = float(mn[ok].mean()) if ok.any() else float("nan")
    if popularity is not None:
        pop = np.asarray(popularity, dtype=np.float64)[filled]
        out["novelty"] = float(np.mean(-np.log2((pop + 1.0) / (n_users + 1.0)))) if filled.size else float("nan")
    return out
