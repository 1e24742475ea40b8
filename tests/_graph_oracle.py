"""numpy restatement of the graph index (recnn_graph_build / recnn_graph_search).

Build, given the k-NN lists N [n, D] (row u: u's D best items, u excluded):
  prune    c_j = #{i < j : N[u, j] is in N[N[u, i]] at a position p < j}; P(u) = N[u] at the first d positions in
           (c_j, j) order
  reverse  every kept edge u -> v at rank r of P(u) makes u a reverse candidate of v, ordered by (r, u)
  merge    v's out-list: P(v)[:d/2], then the reverse candidates, then P(v)[d/2:], skipping ids already present, until
           d are held

Search replay, given a query's keys over every item (tests._exact_retrieval.keys32: bit-exact on small-integer
tables): a buffer of T (key, id, explored) entries sorted by (key, id), starting empty; iteration 0 takes the first
W * d entry points, each later one the out-lists of the W best unexplored entries (marked explored); a candidate
already in the buffer, or repeated within the iteration, is dropped; the buffer becomes the best T of buffer and
candidates.  Stop when nothing is unexplored or after M iterations past iteration 0 (M = 0: no cap)."""
from __future__ import annotations

import numpy as np

NO_ID = 2 ** 31 - 1         # an empty slot: key FLT_MAX, worse than any item
FLT_MAX = float(np.finfo(np.float32).max)


def prune(knn, d):
    """int64 [n, d]: P(u) of every row of knn [n, D] (D >= d)"""
    knn = np.asarray(knn, np.int64)
    n, D = knn.shape
    c = np.zeros((n, D), np.int64)
    i_idx = np.arange(D)[:, None]
    p_idx = np.arange(D)[None, :]
    for u in range(n):
        srt = np.argsort(knn[u], kind="stable")
        sid = knn[u][srt]
        nn = knn[knn[u]]                                    # [D (i), D (p)]: N(v_i)
        at = np.minimum(np.searchsorted(sid, nn), D - 1)
        j = np.where(sid[at] == nn, srt[at], -1)            # the position of N(v_i)[p] in N(u), or -1
        hit = (j >= 0) & (j > i_idx) & (p_idx < j)
        np.add.at(c[u], j[hit], 1)
    order = np.lexsort((np.broadcast_to(np.arange(D), (n, D)), c), axis=1)[:, :d]
    return np.take_along_axis(knn, order, axis=1)


def reverse_merge(P):
    """int64 [n, d]: the out-lists from the pruned lists P [n, d]"""
    P = np.asarray(P, np.int64)
    n, d = P.shape
    u = np.repeat(np.arange(n), d)
    r = np.tile(np.arange(d), n)
    v = P.reshape(-1)
    order = np.lexsort((u, r, v))                          # by v, then r, then u
    vs, us = v[order], u[order]
    starts = np.searchsorted(vs, np.arange(n + 1))
    out = np.empty((n, d), np.int64)
    for x in range(n):
        got = list(P[x, :d // 2])
        have = set(got)
        for y in list(us[starts[x]:starts[x + 1]]) + list(P[x, d // 2:]):
            if len(got) == d:
                break
            if y not in have:
                got.append(int(y))
                have.add(int(y))
        out[x] = got
    return out


def build(knn, d):
    return reverse_merge(prune(knn, d))


def replay(keys, graph, entry, T, W, M=0):
    """(buffer [(key, id)] sorted, iterations past iteration 0) of one query; keys fp32 [n_items]"""
    buf, it, _ = _run(keys, graph, entry, T, W, M)
    return buf, it


def hash_clears(keys, graph, entry, T, W, M=0, hash_fill=2048):
    """the number of times the device's visited hash is cleared during one query's search: it holds every id keyed
    since the last clear, and is cleared and refilled with the buffer's ids before an iteration of nc candidate slots
    could take it past hash_fill ids.  The buffers do not depend on it (see replay)."""
    return _run(keys, graph, entry, T, W, M, hash_fill)[2]


def _run(keys, graph, entry, T, W, M, hash_fill=None):
    keys = np.asarray(keys, np.float32)
    graph = np.asarray(graph, np.int64)
    d = graph.shape[1]
    buf = [(FLT_MAX, NO_ID, True)] * T
    visited, clears = set(), 0

    def merge(cands):
        nonlocal visited, clears
        if hash_fill is not None:
            if len(visited) + len(cands) > hash_fill:
                visited = {i for _, i, _ in buf if i != NO_ID}
                clears += 1
            visited.update(int(c) for c in cands)
        inbuf = {b[1] for b in buf}
        fresh, seen = [], set()
        for c in cands:
            c = int(c)
            if c in inbuf or c in seen:
                continue
            seen.add(c)
            fresh.append((float(keys[c]), c, False))
        return sorted(buf + fresh, key=lambda e: (e[0], e[1]))[:T]

    buf = merge(entry[:min(W * d, len(entry))])
    it = 0
    while not (M > 0 and it >= M):
        parents = [t for t, e in enumerate(buf) if not e[2] and e[1] != NO_ID][:W]
        if not parents:
            break
        for t in parents:
            buf[t] = (buf[t][0], buf[t][1], True)
        buf = merge(np.concatenate([graph[buf[t][1]] for t in parents]))
        it += 1
    return [(k, i) for k, i, _ in buf], it, clears


def search(keys, graph, entry, T, W, M, k, finish, pad, exclude=None, buffers=None):
    """(ids int64 [n_q, k], dist fp32 [n_q, k], iterations [n_q]): the k best eligible entries of each query's final
    buffer, -1 and the distance pad past the last; keys fp32 [n_q, n_items]; finish(row, key array) -> fp32
    distances; exclude: one id list (or None) per query; buffers: the replay() of every query, when already run"""
    keys = np.asarray(keys, np.float32)
    n_q = keys.shape[0]
    if buffers is None:
        buffers = [replay(keys[r], graph, entry, T, W, M) for r in range(n_q)]
    ids = np.full((n_q, k), -1, np.int64)
    kk = np.full((n_q, k), FLT_MAX, np.float32)
    iters = np.array([it for _, it in buffers], np.int64)
    for r, (buf, _) in enumerate(buffers):
        ex = set() if exclude is None or exclude[r] is None else {int(x) for x in exclude[r]}
        got = [(key, i) for key, i in buf if i != NO_ID and i not in ex][:k]
        for t, (key, i) in enumerate(got):
            ids[r, t], kk[r, t] = i, key
    dist = np.stack([finish(r, kk[r]) for r in range(n_q)]).astype(np.float32) if n_q else np.zeros((0, k), np.float32)
    dist[ids < 0] = pad
    return ids, dist, iters


def exact_knn(keys_all, D):
    """int64 [n, D]: row u's D best items by (key, id), u excluded; keys_all fp32 [n, n] (row u = u's keys)"""
    return exact_knn_rows(keys_all, D, 0)


def exact_knn_rows(keys, D, row0):
    """exact_knn for a block of rows row0 .. row0 + len(keys) - 1 of keys fp32 [rows, n]"""
    keys = np.array(keys, np.float32)
    r = np.arange(keys.shape[0])
    keys[r, row0 + r] = np.inf
    return np.argsort(keys, axis=1, kind="stable")[:, :D]
