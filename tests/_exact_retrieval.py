"""Bit-exact restatement of item retrieval (recnn_retrieve_topk / recnn_retrieve_rank, the IVF_FLAT fine scan and the
IVF_PQ refine) for tables and queries of small integers.

When every score <q, t> and every |t|^2 is an integer below 2^11 in magnitude, both GEMM back ends compute the score
exactly (3xTF32: the TF32 hi part is the value, lo = 0; the CUDA-core fp32 FMAs never round), and so does the IVF fine
scan.  The library builds without fast math, so each later fp32 step is one IEEE operation that float32 tensor
arithmetic reproduces bit for bit:

  norms     L2  |t|^2                          COS  1 / max(sqrt(|t|^2), 1e-30)
  keys      L2  fma(-2, s, |t|^2)              IP   -s          COS  -s * (1 / |t|)
  finish    L2  max(key + |q|^2, 0)            IP   -key        COS  -key / max(sqrt(|q|^2), 1e-30)

A key that is NaN or +inf ranks as FLT_MAX: after every finite key, ties by id, and still before an empty slot, so the
item is returned before any -1 pad.  The ids are a stable argsort of the keys; a rank counts the eligible j != t with
(key_j, j) < (key_t, t).  The score is computed in float64 (on the tensors' device), which is exact for these integers.

The non-finite cases of the tests (a row holding 2^64, so |t|^2 overflows; a query holding 2^126, so a score
overflows; NaN rows) keep every finite value exact too: their large values are powers of two times small integers.
They pass bound=None, since the 2^11 bound does not hold for them."""
from __future__ import annotations

import numpy as np
import torch

FLT_MAX = float(np.finfo(np.float32).max)
BOUND = 2 ** 11


def _t(x, device=None):
    t = torch.as_tensor(x)
    return t if device is None else t.to(device)


def scores64(queries, table, bound=BOUND):
    """float64 [n_q, n_items] <q, t>, exact for integer inputs; asserts |s| < bound (None: no check)"""
    s = _t(queries).to(torch.float64) @ _t(table).to(torch.float64).T
    if bound is not None:
        assert bool((s.abs() < bound).all()), "a score is not exact in fp32 on both back ends"
    return s


def norms32(table, metric, bound=BOUND):
    """fp32 [n_items]: recnn_item_norms, |t|^2 (L2) or 1 / |t| (COS); None for IP"""
    if metric == "IP":
        return None
    t = _t(table).to(torch.float64)
    n = (t * t).sum(1)
    if bound is not None:
        assert bool((n.abs() < bound).all()), "a norm is not exact in fp32"
    n = n.to(torch.float32)
    if metric == "L2":
        return n
    # fmaxf ignores a NaN operand: torch.fmax, not torch.maximum
    return torch.ones_like(n) / torch.fmax(torch.sqrt(n), torch.tensor(1e-30, dtype=torch.float32, device=n.device))


def keys32(s64, norms, metric):
    """fp32 keys of a block of float64 scores [n_q, n_items] (smaller is better), NaN and +inf as FLT_MAX"""
    s = s64.to(torch.float32)
    if metric == "L2":
        # fma(-2, s, n): one rounding of the exact value, which float64 holds for fp32 s and n of these magnitudes
        key = (-2.0 * s.to(torch.float64) + norms.to(s64.device).to(torch.float64)[None, :]).to(torch.float32)
    elif metric == "IP":
        key = -s
    else:
        key = -s * norms.to(s64.device)[None, :]
    return finite_key(key)


def finite_key(key):
    """NaN and +inf -> FLT_MAX (fminf(key, FLT_MAX)); -inf stays"""
    return torch.fmin(key, torch.tensor(FLT_MAX, dtype=torch.float32, device=key.device))


def qnorm32(queries):
    q = _t(queries).to(torch.float64)
    return (q * q).sum(1).to(torch.float32)


def finish32(key, qn, metric):
    """fp32 distances of sorted keys [n_q, k] for queries of fp32 |q|^2 qn [n_q]"""
    qn = qn.to(key.device)[:, None]
    if metric == "L2":
        return torch.fmax(key + qn, torch.zeros((), dtype=torch.float32, device=key.device))
    if metric == "COS":
        return -key / torch.fmax(torch.sqrt(qn), torch.tensor(1e-30, dtype=torch.float32, device=key.device))
    return -key


def _eligible(n_items, rows, exclude, device):
    """bool [len(rows), n_items]: False at the excluded ids of each row (exclude: a list of id lists, one per query)"""
    ok = torch.ones(len(rows), n_items, dtype=torch.bool, device=device)
    if exclude is not None:
        for i, r in enumerate(rows):
            ex = torch.as_tensor(np.asarray(exclude[r], np.int64), device=device)
            if ex.numel():
                ok[i, ex] = False
    return ok


def topk(queries, table, metric, k, exclude=None, candidates=None, block=16, bound=BOUND):
    """(ids int64 [n_q, k], dist fp32 [n_q, k]) as numpy: the k smallest (key, id) of the eligible items, -1 and
    FLT_MAX (L2) / -FLT_MAX (IP, COS) past the last eligible one.  candidates: per query an id list (e.g. the union of
    the probed lists), None for every item.  Computed on the tensors' device, `block` queries at a time."""
    q, t = _t(queries), _t(table)
    dev = t.device
    q = q.to(dev)
    n_q, n_items = q.shape[0], t.shape[0]
    norms = norms32(t, metric, bound)
    qn = qnorm32(q)
    ids_out = np.full((n_q, k), -1, np.int64)
    pad = FLT_MAX if metric == "L2" else -FLT_MAX
    dist_out = np.full((n_q, k), pad, np.float32)
    for r0 in range(0, n_q, block):
        rows = range(r0, min(n_q, r0 + block))
        key = keys32(scores64(q[r0:r0 + len(rows)], t, bound), norms, metric)
        ok = _eligible(n_items, rows, exclude, dev)
        if candidates is not None:
            allowed = torch.zeros_like(ok)
            for i, r in enumerate(rows):
                allowed[i, torch.as_tensor(np.asarray(candidates[r], np.int64), device=dev)] = True
            ok &= allowed
        # ineligible items sort after every eligible one (an eligible key is at most FLT_MAX): +inf and a flag
        key = torch.where(ok, key, torch.full_like(key, float("inf")))
        order = torch.sort(key, dim=1, stable=True).indices[:, :k]
        keep = torch.gather(ok, 1, order)
        fin = finish32(torch.gather(key, 1, order), qn[r0:r0 + len(rows)], metric)
        order, keep, fin = order.cpu().numpy(), keep.cpu().numpy(), fin.cpu().numpy()
        for i, r in enumerate(rows):
            n = int(keep[i].sum())                              # eligible items come first, so keep is a prefix
            assert keep[i, :n].all()
            ids_out[r, :n] = order[i, :n]
            dist_out[r, :n] = fin[i, :n]
    return ids_out, dist_out


def rank(queries, table, metric, target, exclude=None, block=16, bound=BOUND):
    """int64 [n_q] numpy: the number of eligible j != target with (key_j, j) < (key_t, t); a target is never
    excluded"""
    q, t = _t(queries), _t(table)
    dev = t.device
    q = q.to(dev)
    n_q, n_items = q.shape[0], t.shape[0]
    target = torch.as_tensor(np.asarray(target, np.int64), device=dev)
    norms = norms32(t, metric, bound)
    ids = torch.arange(n_items, device=dev)
    out = np.empty(n_q, np.int64)
    for r0 in range(0, n_q, block):
        rows = range(r0, min(n_q, r0 + block))
        key = keys32(scores64(q[r0:r0 + len(rows)], t, bound), norms, metric)
        tg = target[r0:r0 + len(rows)]
        kt = torch.gather(key, 1, tg[:, None])
        beats = (key < kt) | ((key == kt) & (ids[None, :] < tg[:, None]))
        beats &= _eligible(n_items, rows, exclude, dev)
        beats &= ids[None, :] != tg[:, None]
        out[r0:r0 + len(rows)] = beats.sum(1).cpu().numpy()
    return out


def small_ints(rng, shape, lo=-3, hi=3):
    """fp32 integers uniform in [lo, hi]"""
    return rng.integers(lo, hi + 1, size=shape).astype(np.float32)
