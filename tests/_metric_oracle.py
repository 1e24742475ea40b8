"""Restatement of the retrieval metrics that are not inner products (RECNN_METRIC_L1 .. RECNN_METRIC_CORR, recnn_b200.h)
and of the scipy.spatial.distance names ItemIndex serves.

``dist32`` replays the kernel in float32, one IEEE operation per step and d ascending, so for L1, LINF, CANBERRA and
BRAYCURTIS it is bit for bit what the device computes, on any inputs:

  L1          acc += |q_d - t_d|
  LINF        acc = max(acc, |q_d - t_d|)                       NaN-propagating (torch.maximum)
  CANBERRA    acc += den == 0 ? 0 : |q_d - t_d| / den,  den = |q_d| + |t_d|
  BRAYCURTIS  num += |q_d - t_d|, den += |q_d + t_d|;  num == 0 ? 0 : num / den
  CORR        1 - dot / (|q_c| |t_c|) clipped to [0, 2] (NaN kept), 1 when |q_c| |t_c| == 0; a constant row has mean x_0
              and centred norm 0

CORR's replay rounds each fma through float64 (an fma up to a double rounding), so it is not bit-exact: the device
result is held to ``dist64`` within ``corr_bar``.  ``dist64`` states every metric in float64 with the same conventions.
The key of a distance is the distance, NaN and +inf as FLT_MAX; ids are a stable argsort of the keys."""
from __future__ import annotations

import numpy as np
import torch

FLT_MAX = float(np.finfo(np.float32).max)
U32 = 2.0 ** -24
EXACT = ("L1", "LINF", "CANBERRA", "BRAYCURTIS")
CODES = EXACT + ("CORR",)
# ItemIndex names of the codes, and the scipy.spatial.distance function of every name the index serves
NAME = {"L1": "cityblock", "LINF": "chebyshev", "CANBERRA": "canberra", "BRAYCURTIS": "braycurtis",
        "CORR": "correlation"}
SCIPY_NAMES = ("euclidean", "cosine", "correlation", "canberra", "minkowski", "chebyshev", "braycurtis", "cityblock")


def _t(x, device=None):
    t = torch.as_tensor(x)
    return t if device is None else t.to(device)


def corr_stats32(x):
    """(mean, centred norm) fp32 [n] of the rows of x [n, dim], as recnn_item_norms(CORR) and the kernel's query
    staging compute them: the mean is the ascending fp32 sum over dim, the norm sqrt of the fma-sum of squares"""
    x = _t(x).to(torch.float32)
    dim = x.shape[1]
    s = torch.zeros(x.shape[0], dtype=torch.float32, device=x.device)
    for d in range(dim):
        s = s + x[:, d]
    mean = s / torch.full_like(s, float(dim))                   # a tensor divisor: torch multiplies by 1 / scalar
    n = torch.zeros_like(s)
    for d in range(dim):
        c = x[:, d] - mean
        n = (n.double() + c.double() * c.double()).float()
    const = (x == x[:, :1]).all(1)
    mean = torch.where(const, x[:, 0], mean)
    n = torch.where(const, torch.zeros_like(n), torch.sqrt(n))
    return mean, n


def dist32(queries, table, code):
    """fp32 [n_q, n_items]: the kernel's distance of every pair (not yet a key), on the tensors' device"""
    q, t = _t(queries).to(torch.float32), _t(table).to(torch.float32)
    t = t.to(q.device)
    dim = q.shape[1]
    zero = torch.zeros((), dtype=torch.float32, device=q.device)
    if code == "CORR":
        qm, qn = corr_stats32(q)
        tm, tn = corr_stats32(t)
        q, t = q - qm[:, None], t - tm[:, None]
    a = torch.zeros(q.shape[0], t.shape[0], dtype=torch.float32, device=q.device)
    b = torch.zeros_like(a)
    for d in range(dim):
        qd, td = q[:, d:d + 1], t[None, :, d]
        if code == "L1":
            a = a + (qd - td).abs()
        elif code == "LINF":
            a = torch.maximum(a, (qd - td).abs())
        elif code == "CANBERRA":
            den = qd.abs() + td.abs()
            a = a + torch.where(den == 0, zero, (qd - td).abs() / den)
        elif code == "BRAYCURTIS":
            a = a + (qd - td).abs()
            b = b + (qd + td).abs()
        else:
            a = (a.double() + qd.double() * td.double()).float()
    if code == "BRAYCURTIS":
        return torch.where(a == 0, zero, a / b)
    if code == "CORR":
        den = qn[:, None] * tn[None, :]
        r = torch.where(den == 0, zero, a / den)
        d = 1.0 - r
        d = torch.where(d < 0, zero, d)
        return torch.where(d > 2, torch.full_like(d, 2.0), d)
    return a


def dist64(queries, table, code):
    """float64 [n_q, n_items]: the same metrics with the same conventions, computed in float64"""
    q, t = _t(queries).to(torch.float64), _t(table).to(torch.float64)
    t = t.to(q.device)
    diff = (q[:, None, :] - t[None, :, :]).abs() if code != "CORR" else None
    if code == "L1":
        return diff.sum(2)
    if code == "LINF":
        return diff.amax(2) if diff.shape[2] else diff.sum(2)
    if code == "CANBERRA":
        den = q.abs()[:, None, :] + t.abs()[None, :, :]
        return torch.where(den == 0, torch.zeros_like(den), diff / den).sum(2)
    if code == "BRAYCURTIS":
        num, den = diff.sum(2), (q[:, None, :] + t[None, :, :]).abs().sum(2)
        return torch.where(num == 0, torch.zeros_like(num), num / den)
    qc, tc = q - q.mean(1, keepdim=True), t - t.mean(1, keepdim=True)
    qconst, tconst = (q == q[:, :1]).all(1), (t == t[:, :1]).all(1)
    qc[qconst], tc[tconst] = 0.0, 0.0
    den = qc.norm(dim=1)[:, None] * tc.norm(dim=1)[None, :]
    r = torch.where(den == 0, torch.zeros_like(den), (qc @ tc.T) / den)
    return (1.0 - r).clamp(0.0, 2.0)


def corr_bar(queries, table):
    """float64 [n_q, n_items]: a bound on |fp32 CORR - float64 CORR| of each pair.  The fp32 mean is off by at most
    about u (sum |x| + |mean|) (sequential sum, then a division); a centred value inherits that error plus one
    rounding, the fma dot adds (dim + 2) u |q_c| |t_c| by Cauchy-Schwarz, each norm about (dim + 2) u / 2 of itself,
    and the division and the 1 - r one u each.  The bar doubles the sum."""
    q, t = _t(queries).to(torch.float64), _t(table).to(torch.float64)
    t = t.to(q.device)
    dim = q.shape[1]

    def rel(x):
        c = x - x.mean(1, keepdim=True)
        n = c.norm(dim=1)
        dmu = U32 * (x.abs().sum(1) + x.mean(1).abs())
        return torch.where(n > 0, np.sqrt(dim) * dmu / n, torch.zeros_like(n))

    e = (2 * dim + 8) * U32 + 2 * (rel(q)[:, None] + rel(t)[None, :])
    return 2.0 * e


def finite_key(d):
    return torch.fmin(d, torch.tensor(FLT_MAX, dtype=d.dtype, device=d.device))


def _eligible(n_items, rows, exclude, device):
    ok = torch.ones(len(rows), n_items, dtype=torch.bool, device=device)
    if exclude is not None:
        for i, r in enumerate(rows):
            ex = torch.as_tensor(np.asarray(exclude[r], np.int64), device=device)
            if ex.numel():
                ok[i, ex] = False
    return ok


def topk(queries, table, code, k, exclude=None, block=64):
    """(ids int64 [n_q, k], dist fp32 [n_q, k]) numpy: the stable argsort of the replay's keys over the eligible items
    (exclude: one id list per query), -1 and FLT_MAX past the last eligible one"""
    q, t = _t(queries).to(torch.float32), _t(table).to(torch.float32)
    dev = t.device
    q = q.to(dev)
    n_q, n_items = q.shape[0], t.shape[0]
    ids_out = np.full((n_q, k), -1, np.int64)
    dist_out = np.full((n_q, k), FLT_MAX, np.float32)
    for r0 in range(0, n_q, block):
        rows = range(r0, min(n_q, r0 + block))
        key = finite_key(dist32(q[r0:r0 + len(rows)], t, code))
        ok = _eligible(n_items, rows, exclude, dev)
        key = torch.where(ok, key, torch.full_like(key, float("inf")))
        order = torch.sort(key, dim=1, stable=True).indices[:, :k]
        keep = torch.gather(ok, 1, order).cpu().numpy()
        kd = torch.gather(key, 1, order).cpu().numpy()
        order = order.cpu().numpy()
        for i, r in enumerate(rows):
            n = int(keep[i].sum())
            ids_out[r, :n] = order[i, :n]
            dist_out[r, :n] = kd[i, :n]
    return ids_out, dist_out


def rank(queries, table, code, target, exclude=None, block=64):
    """int64 [n_q] numpy: the eligible j != target whose (key, j) beats (key_t, target)"""
    q, t = _t(queries).to(torch.float32), _t(table).to(torch.float32)
    dev = t.device
    q = q.to(dev)
    n_q, n_items = q.shape[0], t.shape[0]
    target = torch.as_tensor(np.asarray(target, np.int64), device=dev)
    ids = torch.arange(n_items, device=dev)
    out = np.empty(n_q, np.int64)
    for r0 in range(0, n_q, block):
        rows = range(r0, min(n_q, r0 + block))
        key = finite_key(dist32(q[r0:r0 + len(rows)], t, code))
        tg = target[r0:r0 + len(rows)]
        kt = torch.gather(key, 1, tg[:, None])
        beats = (key < kt) | ((key == kt) & (ids[None, :] < tg[:, None]))
        beats &= _eligible(n_items, rows, exclude, dev) & (ids[None, :] != tg[:, None])
        out[r0:r0 + len(rows)] = beats.sum(1).cpu().numpy()
    return out


def scipy_dist(queries, table, name, p=None):
    """float64 [n_q, n_items] numpy: scipy.spatial.distance.cdist under a name the index serves"""
    from scipy.spatial.distance import cdist
    q, t = np.asarray(_t(queries).cpu(), np.float64), np.asarray(_t(table).cpu(), np.float64)
    if name == "minkowski":
        return cdist(q, t, "minkowski", p=2 if p is None else p)
    return cdist(q, t, name)


def small_ints(rng, shape, lo=-3, hi=3):
    """fp32 integers uniform in [lo, hi]"""
    return rng.integers(lo, hi + 1, size=shape).astype(np.float32)


def name_dist32(queries, table, name, p=None):
    """fp32 [n_q, n_items] numpy: the distance ItemIndex(table, name, p) reports for every item.  euclidean and cosine
    run on L2 / COS (tests/_exact_retrieval.py, exact when the scores are integers below 2^11) and convert; the others
    are dist32 of their code, NaN and +inf as FLT_MAX."""
    from tests import _exact_retrieval as X
    if name == "minkowski":
        name = {1: "cityblock", 2: "euclidean", float("inf"): "chebyshev"}[2 if p is None else p]
    q, t = _t(queries).to(torch.float32), _t(table).to(torch.float32)
    if name in ("euclidean", "cosine"):
        metric = "L2" if name == "euclidean" else "COS"
        key = X.keys32(X.scores64(q, t, None), X.norms32(t, metric, None), metric)
        d = X.finish32(key, X.qnorm32(q), metric)
        d = torch.sqrt(d) if name == "euclidean" else torch.clamp(1.0 - d, 0.0, 2.0)
        return d.cpu().numpy()
    code = {v: k for k, v in NAME.items()}[name]
    return finite_key(dist32(q, t, code)).cpu().numpy()
