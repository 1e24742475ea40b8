"""Nearest-item retrieval over the embedding table (recnn/data/db_con.py:45-56,
examples/streamlit_demo.py:189-215).

The reference hands the actor's generated action to an external vector index (a
Milvus server, or faiss IndexFlatL2 / IndexFlatIP in the demo) and gets back
``topk`` item ids and distances.  Here the index IS the embedding table that is
already resident in HBM for the update step: ``search`` is one exact
``[n, dim] x [dim, n_items]`` contraction on the tensor cores plus an exact
top-k, both in librecnn_b200.so (recnn_retrieve_topk).  No server, no CPU path.

``ItemIndex(table, metric).search(vecs, topk)`` returns a ``SearchResult`` with
the reference's accessors ``.id(device)`` / ``.dist(device)``; ``exclude=`` an
``ItemSets`` (recnn_b200/data/item_sets.py) keeps each query's set out of its
results (recnn_retrieve_topk_sets).
``MilvusConnection(env, ...)`` keeps the reference's constructor shape for code
written against recnn.data.db_con.
"""
from __future__ import annotations

import torch

from .. import _lib

_METRICS = {"L2": _lib.METRIC_L2, "IP": _lib.METRIC_IP, "COS": _lib.METRIC_COS}


class SearchResult:
    """recnn/data/db_con.py:5-13: ids int64 [n, topk] and distances fp32 [n, topk], best first."""

    def __init__(self, ids, dist):
        self.ids, self.distances = ids, dist

    def id(self, device=None):
        return self.ids if device is None else self.ids.to(device)

    def dist(self, device=None):
        return self.distances if device is None else self.distances.to(device)


class ItemIndex:
    """Exact top-k search over an item-embedding matrix resident on one GPU.

    metric: "L2" (squared Euclidean distance, smallest first -- faiss IndexFlatL2 / Milvus L2),
            "IP" (inner product, largest first), "COS" (cosine similarity, largest first).
    """

    def __init__(self, embeddings, metric="L2"):
        if metric not in _METRICS:
            raise ValueError("metric must be one of %s" % sorted(_METRICS))
        if not torch.is_tensor(embeddings):
            embeddings = torch.as_tensor(embeddings)
        if embeddings.device.type != "cuda":
            raise _lib.RecnnError("ItemIndex needs the embedding table on a CUDA device (got %s); there is no CPU path"
                                  % embeddings.device)
        self.table = embeddings.detach().to(torch.float32).contiguous()
        self.metric_name, self.metric = metric, _METRICS[metric]
        self.device = self.table.device
        self.n_items, self.dim = int(self.table.shape[0]), int(self.table.shape[1])
        self.norms = None
        if self.metric != _lib.METRIC_IP:
            self.norms = torch.empty(self.n_items, dtype=torch.float32, device=self.device)
            with torch.cuda.device(self.device):
                _lib.check(_lib.lib().recnn_item_norms(self.table.data_ptr(), self.n_items, self.dim, self.metric,
                                                       self.norms.data_ptr(), _lib.stream_ptr(self.device)))
        self._ws = None

    def search(self, search_vecs, topk=10, search_param=None, exclude=None, exclude_rows=None):
        """search_vecs: [n, dim] (tensor / array on any device).  Returns SearchResult on the index's device.
        ``exclude``: an ``ItemSets`` of item ids never returned (e.g. ``DeviceFrameFeed.seen_items()``), with
        ``exclude_rows`` int64 [n] naming each query's set (-1: none; default query r -> set r).  A query with fewer
        than topk eligible items ends in id -1, distance FLT_MAX (L2) or -FLT_MAX (IP, COS).  An excluded id outside
        [0, n_items) raises IndexError, a malformed table ValueError."""
        from .item_sets import ItemSets, row_map
        q = torch.as_tensor(search_vecs)
        if q.dim() == 1:
            q = q.unsqueeze(0)
        if q.dim() != 2 or q.shape[1] != self.dim:
            raise ValueError("search_vecs must be [n, %d]" % self.dim)
        topk = int(topk)
        if not 1 <= topk <= min(64, self.n_items):
            raise ValueError("topk must be in [1, min(64, n_items)]")
        n = int(q.shape[0])
        sets = rows = None
        if exclude is not None:
            if not isinstance(exclude, ItemSets):
                raise ValueError("exclude must be a recnn_b200.data.ItemSets (got %s)" % type(exclude).__name__)
            sets, rows = row_map(exclude, exclude_rows, n)
        elif exclude_rows is not None:
            raise ValueError("exclude_rows maps queries to the sets of an ItemSets exclude")
        q = q.detach().to(device=self.device, dtype=torch.float32).contiguous()
        ids = torch.empty(n, topk, dtype=torch.int64, device=self.device)
        dist = torch.empty(n, topk, dtype=torch.float32, device=self.device)
        if n == 0:
            return SearchResult(ids, dist)
        L = _lib.lib()
        need = L.recnn_retrieve_workspace_bytes(n, self.n_items, topk)
        if self._ws is None or self._ws.numel() < need:
            self._ws = torch.empty(need, dtype=torch.uint8, device=self.device)
        args = (q.data_ptr(), n, self.dim, self.table.data_ptr(), self.n_items, _lib.ptr(self.norms), self.metric, topk)
        with torch.cuda.device(self.device):
            if sets is None:
                _lib.check(L.recnn_retrieve_topk(*args, ids.data_ptr(), dist.data_ptr(), self._ws.data_ptr(),
                                                 self._ws.numel(), _lib.stream_ptr(self.device)))
                return SearchResult(ids, dist)
            sets = sets.to(self.device)
            rows = None if rows is None else rows.to(self.device).contiguous()
            flag = torch.empty(1, dtype=torch.int32, device=self.device)
            _lib.check(L.recnn_retrieve_topk_sets(*args, sets.ids.data_ptr() if sets.ids.numel() else None,
                                                  sets.ids.numel(), sets.offsets.data_ptr(), len(sets),
                                                  _lib.ptr(rows), ids.data_ptr(), dist.data_ptr(), flag.data_ptr(),
                                                  self._ws.data_ptr(), self._ws.numel(),
                                                  _lib.stream_ptr(self.device)))
        bits = int(flag.item())
        if bits & 1:
            raise IndexError("an excluded item id is out of range for the index's %d items" % self.n_items)
        if bits & 4:
            raise ValueError("malformed exclusion table: a set is not ascending, its offsets are out of range or "
                             "decreasing, or an exclude_rows entry is outside [-1, %d)" % len(sets))
        return SearchResult(ids, dist)

    def rank(self, search_vecs, target, exclude=None, exclude_rows=None):
        """int64 [n]: for offline evaluation, the number of items ``search`` on the same queries would return before
        ``target[q]`` (better key, equal keys the smaller id), i.e. the target's position in ``search(vecs, k)`` when
        below k and the target is absent otherwise, at any k.  ``exclude`` / ``exclude_rows`` as in ``search``; a
        query's target is never excluded.  DDPG / TD3: ``index.rank(actor(state), target, ...)``.  A target or
        excluded id outside [0, n_items) raises IndexError, a malformed table ValueError."""
        from .item_sets import ItemSets, row_map
        q = torch.as_tensor(search_vecs)
        if q.dim() == 1:
            q = q.unsqueeze(0)
        if q.dim() != 2 or q.shape[1] != self.dim:
            raise ValueError("search_vecs must be [n, %d]" % self.dim)
        n = int(q.shape[0])
        if (not torch.is_tensor(target) or target.dim() != 1 or target.shape[0] != n
                or target.dtype.is_floating_point or target.dtype.is_complex or target.dtype == torch.bool):
            raise ValueError("target must be an integer tensor [n] with n = %d queries (got %s)"
                             % (n, "%s %s" % (tuple(target.shape), target.dtype) if torch.is_tensor(target)
                                else type(target).__name__))
        sets = rows = None
        if exclude is not None:
            if not isinstance(exclude, ItemSets):
                raise ValueError("exclude must be a recnn_b200.data.ItemSets (got %s)" % type(exclude).__name__)
            sets, rows = row_map(exclude, exclude_rows, n)
        elif exclude_rows is not None:
            raise ValueError("exclude_rows maps queries to the sets of an ItemSets exclude")
        q = q.detach().to(device=self.device, dtype=torch.float32).contiguous()
        rank = torch.empty(n, dtype=torch.int64, device=self.device)
        if n == 0:
            return rank
        target = target.detach().to(device=self.device, dtype=torch.int64).contiguous()
        L = _lib.lib()
        need = L.recnn_retrieve_rank_workspace_bytes(n, self.n_items)
        if self._ws is None or self._ws.numel() < need:
            self._ws = torch.empty(need, dtype=torch.uint8, device=self.device)
        args = (q.data_ptr(), n, self.dim, self.table.data_ptr(), self.n_items, _lib.ptr(self.norms), self.metric,
                target.data_ptr())
        flag = torch.empty(1, dtype=torch.int32, device=self.device)
        with torch.cuda.device(self.device):
            if sets is None:
                _lib.check(L.recnn_retrieve_rank(*args, rank.data_ptr(), flag.data_ptr(), self._ws.data_ptr(),
                                                 self._ws.numel(), _lib.stream_ptr(self.device)))
            else:
                sets = sets.to(self.device)
                rows = None if rows is None else rows.to(self.device).contiguous()
                _lib.check(L.recnn_retrieve_rank_sets(*args, sets.ids.data_ptr() if sets.ids.numel() else None,
                                                      sets.ids.numel(), sets.offsets.data_ptr(), len(sets),
                                                      _lib.ptr(rows), rank.data_ptr(), flag.data_ptr(),
                                                      self._ws.data_ptr(), self._ws.numel(),
                                                      _lib.stream_ptr(self.device)))
        bits = int(flag.item())
        if bits & 1:
            raise IndexError("a target or excluded item id is out of range for the index's %d items" % self.n_items)
        if bits & 4:
            raise ValueError("malformed exclusion table: a set is not ascending, its offsets are out of range or "
                             "decreasing, or an exclude_rows entry is outside [-1, %d)" % len(sets))
        return rank


class MilvusConnection(ItemIndex):
    """Constructor shape of recnn.data.db_con.MilvusConnection(env, name=..., port=..., param=...): the collection
    is ``env.base.embeddings``; ``param["metric_type"]`` may be "L2" (default) or "IP".  No Milvus server is involved."""

    def __init__(self, env, name="movies_L2", port="19530", param=None):
        metric = "L2"
        if param and "metric_type" in param:
            mt = str(param["metric_type"]).upper()
            metric = "IP" if mt.endswith("IP") else "L2"
        emb = env.base.embeddings if hasattr(env, "base") else env
        super().__init__(emb, metric)
        self.name = name
        self.statuses = {}

    def get_log(self):
        return self.statuses
