"""Float64 restatement of IVF_PQ's codes and ADC search (recnn_ivf_pq_build / recnn_ivf_pq_search, DESIGN.md 4c-ivfpq).

The coarse lists are IVF_FLAT's (tests/_ivf_oracle.py).  An item x in list l is stored as m codes of its residual
r = x - c_l (COS: x the unit row); its reconstruction is c_l + [B_0[code_0], ..., B_{m-1}[code_{m-1}]].  adc_values()
computes the ADC keys through the lookup tables the device builds, reconstruction_values() the same quantity directly;
probed_topk() is the top-k over the union of given lists under those values."""
from __future__ import annotations

import numpy as np
import torch

from tests import _ivf_oracle as V

CODEWORDS = 256
TRAIN_MAX = 65536


def pq_sample_plan(n_sample, seed=0):
    """the positions of the initial codewords among the first min(n_sample, 65536) sample points"""
    g = torch.Generator().manual_seed(int(seed) + 1)
    return torch.randperm(min(n_sample, TRAIN_MAX), generator=g)[:CODEWORDS].numpy().astype(np.int64)


def item_lists(offsets, n_items, ids):
    """[n_items] the list of each item"""
    out = np.empty(n_items, np.int64)
    out[ids] = np.repeat(np.arange(len(offsets) - 1), np.diff(offsets))
    return out


def residuals(table, metric, centroids, offsets, ids):
    """[n_items, dim] float64 residual of every item (by item id) from its list's centroid"""
    t = np.asarray(table, np.float64)
    if metric == "COS":
        t = V._unit(t)
    return t - np.asarray(centroids, np.float64)[item_lists(offsets, len(t), ids)]


def encode(res, codebooks):
    """[n, m] the nearest codeword of each subvector (float64, ties to the smaller code) and the [n, m, 256] distances"""
    b = np.asarray(codebooks, np.float64)
    m, _, dsub = b.shape
    r = np.asarray(res, np.float64).reshape(len(res), m, dsub)
    d = ((r[:, :, None, :] - b[None]) ** 2).sum(-1)
    return np.argmin(d, axis=2), d


def reconstructions(centroids, codebooks, codes_by_item, item_list):
    """[n_items, dim] float64 c_list + the codewords of each item's codes"""
    b = np.asarray(codebooks, np.float64)
    m = b.shape[0]
    parts = b[np.arange(m)[None, :], np.asarray(codes_by_item, np.int64)]       # [n, m, dsub]
    return np.asarray(centroids, np.float64)[item_list] + parts.reshape(len(parts), -1)


def reconstruction_values(queries, rec, metric):
    """[n, n_items] L2 squared distance, IP inner product, COS unit query . reconstruction (not renormalised)"""
    q = np.asarray(queries, np.float64)
    if metric == "L2":
        return (q * q).sum(1)[:, None] + (rec * rec).sum(1)[None, :] - 2.0 * q @ rec.T
    if metric == "COS":
        q = V._unit(q)
    return q @ rec.T


def adc_values(queries, metric, centroids, codebooks, codes_by_item, item_list):
    """[n, n_items] the same values through lookup tables: L2 sum_j LUT_{q,l}[j][code_j] with LUT_{q,l}[j][c] =
    |q_j - c_l,j - B_j[c]|^2; IP / COS <q, c_l> + sum_j <q_j, B_j[code_j]>"""
    q = np.asarray(queries, np.float64)
    if metric == "COS":
        q = V._unit(q)
    c = np.asarray(centroids, np.float64)
    b = np.asarray(codebooks, np.float64)
    m, _, dsub = b.shape
    codes = np.asarray(codes_by_item, np.int64)
    out = np.empty((len(q), len(codes)))
    for i in range(len(q)):
        qj = q[i].reshape(m, dsub)
        if metric == "L2":
            rq = q[i][None, :] - c                                               # [nlist, dim]
            lut = ((rq.reshape(len(c), m, 1, dsub) - b[None]) ** 2).sum(-1)      # [nlist, m, 256]
            out[i] = lut[item_list[:, None], np.arange(m)[None, :], codes].sum(1)
        else:
            lut = (qj[:, None, :] * b).sum(-1)                                   # [m, 256]
            out[i] = (c @ q[i])[item_list] + lut[np.arange(m)[None, :], codes].sum(1)
    return out


def probed_topk(values, metric, probes, offsets, ids, k, exclude=None):
    """top-k over the union of each query's probed lists (minus its exclude set) under values [n, n_items] (L2 smallest
    first, IP / COS largest first, ties to the smaller id): ids int64 [n, k] (-1 pad), values float64 (NaN on pads)"""
    n = len(values)
    out_i = np.full((n, k), -1, np.int64)
    out_d = np.full((n, k), np.nan)
    for r in range(n):
        cand = np.sort(np.concatenate([ids[offsets[l]:offsets[l + 1]] for l in probes[r]]))
        if exclude is not None and exclude[r] is not None:
            cand = np.setdiff1d(cand, np.asarray(exclude[r], np.int64))
        v = values[r, cand]
        key = v if metric == "L2" else -v
        order = np.lexsort((cand, key))[:k]
        out_i[r, :len(order)] = cand[order]
        out_d[r, :len(order)] = v[order]
    return out_i, out_d
