"""Float64 restatement of the IVF_FLAT index (recnn_ivf_build / recnn_ivf_search, DESIGN.md 4c-ivf).

build() replays the device build: the seeded sample and init, Lloyd rounds (nearest centroid in L2, ties to the
smaller id; the mean of the members; faiss's split of empty lists with the largest-count donor; COS on unit rows with
renormalised centroids), then the final CSR.  probed_topk() is the exact top-k over the union of given lists."""
from __future__ import annotations

import numpy as np
import torch

from oracle import recnn_oracle as O

EPS = 1.0 / 1024.0


def sample_plan(n_items, nlist, seed=0, max_points_per_centroid=256):
    """(sample, init) as numpy int64: every item, or the first nlist * mppc of a seeded randperm; init the first nlist
    of a second randperm of the sample from the same generator"""
    g = torch.Generator().manual_seed(int(seed))
    cap = nlist * max_points_per_centroid
    sample = torch.randperm(n_items, generator=g)[:cap] if n_items > cap else torch.arange(n_items)
    init = torch.randperm(len(sample), generator=g)[:nlist]
    return sample.numpy().astype(np.int64), init.numpy().astype(np.int64)


def _unit(x):
    return x / np.maximum(np.linalg.norm(x, axis=1, keepdims=True), 1e-30)


def l2_keys(x, c):
    """[n, nlist] float64 squared distances"""
    return (x * x).sum(1)[:, None] + (c * c).sum(1)[None, :] - 2.0 * (x @ c.T)


def assign(x, c):
    """nearest centroid in L2, ties to the smaller id (argmin keeps the first)"""
    return np.argmin(l2_keys(x, c), axis=1)


def split_empty(c, counts):
    """faiss's split with the largest-count donor (ties: smaller id), in ascending id of the empty lists; in place.
    Returns the (empty, donor) pairs."""
    sign = np.where(np.arange(c.shape[1]) % 2 == 0, 1.0, -1.0)
    pairs = []
    for i in range(len(counts)):
        if counts[i] != 0:
            continue
        j = int(np.argmax(counts))            # first maximum: the smaller id
        v = c[j].copy()
        c[i] = v * (1.0 + sign * EPS)
        c[j] = v * (1.0 - sign * EPS)
        half = counts[j] * 0.5
        counts[i], counts[j] = half, counts[j] - half
        pairs.append((i, j))
    return pairs


def lloyd(x, init_centroids, n_iter, spherical):
    """n_iter rounds from the given centroids over the training points x (unit rows when spherical)"""
    c = np.array(init_centroids, dtype=np.float64)
    for _ in range(n_iter):
        a = assign(x, c)
        counts = np.bincount(a, minlength=len(c)).astype(np.float64)
        for l in np.nonzero(counts)[0]:
            c[l] = x[a == l].mean(0)
        split_empty(c, counts)
        if spherical:
            c = _unit(c)
    return c


def final_lists(table, metric, c):
    """(list_offsets, list_ids, item_list): every item to its nearest centroid (COS: largest cosine)"""
    t = np.asarray(table, np.float64)
    if metric == "COS":
        a = np.argmax(_unit(t) @ _unit(c).T, axis=1)
    else:
        a = assign(t, c)
    ids = np.argsort(a, kind="stable").astype(np.int64)
    offsets = np.concatenate([[0], np.cumsum(np.bincount(a, minlength=len(c)))]).astype(np.int64)
    return offsets, ids, a


def build(table, metric, nlist, n_iter=25, seed=0, max_points_per_centroid=256):
    """-> (centroids float64 [nlist, dim], list_offsets, list_ids)"""
    t = np.asarray(table, np.float64)
    sample, init = sample_plan(len(t), nlist, seed, max_points_per_centroid)
    x = t[sample]
    if metric == "COS":
        x = _unit(x)
    c = lloyd(x, x[init], n_iter, metric == "COS")
    offsets, ids, _ = final_lists(t, metric, c)
    return c, offsets, ids


def coarse(queries, centroids, metric, nprobe):
    """each query's nprobe best lists under the metric, as recnn_retrieve_topk ranks them"""
    return O.retrieve_topk(queries, centroids, nprobe, metric)[0]


def probed_topk(queries, table, metric, probes, offsets, ids, k, exclude=None):
    """exact top-k over the union of each query's probed lists (minus its exclude set): ids int64 [n, k] (-1 pad),
    values float64 [n, k] as recnn_retrieve_topk reports them (NaN on pads)"""
    q = np.asarray(queries, np.float64)
    t = np.asarray(table, np.float64)
    n = len(q)
    out_i = np.full((n, k), -1, np.int64)
    out_d = np.full((n, k), np.nan)
    for r in range(n):
        cand = np.sort(np.concatenate([ids[offsets[l]:offsets[l + 1]] for l in probes[r]]))
        if exclude is not None and exclude[r] is not None:
            cand = np.setdiff1d(cand, np.asarray(exclude[r], np.int64))
        if len(cand) == 0:
            continue
        i, d = O.retrieve_topk(q[r:r + 1], t[cand], min(k, len(cand)), metric)
        out_i[r, :i.shape[1]] = cand[i[0]]
        out_d[r, :i.shape[1]] = d[0]
    return out_i, out_d


def blobs(n_per, centers, scale, seed):
    """points around each center (n_per each, in blob order) and their blob labels"""
    rng = np.random.default_rng(seed)
    centers = np.asarray(centers, np.float64)
    x = np.concatenate([c + scale * rng.standard_normal((n_per, centers.shape[1])) for c in centers])
    return x, np.repeat(np.arange(len(centers)), n_per)
