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

``ItemIndex.build_ivf(nlist)`` adds an inverted-file index (IVF_FLAT, as Milvus
and faiss name it), built on the device: k-means lists over the table, after
which ``search(..., search_param={"nprobe": p})`` scans only the lists of each
query's p nearest centroids (recnn_ivf_build / recnn_ivf_search).  ``rank``
stays exact, so recall can be measured against it or against a flat index.
``build_ivf(nlist, m=M)`` builds IVF_PQ instead: the same lists, each item
stored as M one-byte codes of its residual, scanned through lookup tables and
optionally re-ranked exactly from the table (``search_param={"refine": r}``).

``ItemIndex.build_graph()`` adds a proximity-graph index instead (CAGRA-style,
Milvus's GPU_CAGRA): a pruned k-NN graph of the items, built on the device,
after which ``search(..., search_param={"itopk_size": T, "search_width": W,
"max_iterations": M})`` runs a beam search with one CTA per query
(recnn_graph_build / recnn_graph_search).  An index holds at most one of the
IVF and graph indexes.

``ItemIndex`` also takes the eight ``scipy.spatial.distance`` names the reference
demo ranks by (examples/streamlit_demo.py:207-230, 319-345), so that its
``rank(action, distance.<name>, k)`` is ``ItemIndex(table, name).search(action, k)``:
"euclidean" and "cosine" run on L2 and COS, "cityblock", "chebyshev",
"canberra", "braycurtis" and "correlation" on CUDA-core distance kernels
(recnn_b200.h documents their fp32 arithmetic), "minkowski" on one of them by p.
"""
from __future__ import annotations

import ctypes
from typing import NamedTuple

import torch

from .. import _lib

_METRICS = {"L2": _lib.METRIC_L2, "IP": _lib.METRIC_IP, "COS": _lib.METRIC_COS}
# scipy.spatial.distance names -> the metric that ranks them; "euclidean" reports sqrt of L2's squared distance and
# "cosine" 1 - COS's similarity, the others report the kernel's distance as it is
_SCIPY = {"euclidean": _lib.METRIC_L2, "cosine": _lib.METRIC_COS, "cityblock": _lib.METRIC_L1,
          "chebyshev": _lib.METRIC_LINF, "canberra": _lib.METRIC_CANBERRA, "braycurtis": _lib.METRIC_BRAYCURTIS,
          "correlation": _lib.METRIC_CORR}
_MINKOWSKI = {1.0: "cityblock", 2.0: "euclidean", float("inf"): "chebyshev"}
_FLT_MAX = float(torch.finfo(torch.float32).max)


def _metric_name(metric, p):
    """the name in _METRICS or _SCIPY that metric (and minkowski's p) stands for"""
    if metric == "minkowski":
        p = 2.0 if p is None else float(p)
        if p not in _MINKOWSKI:
            raise ValueError("minkowski is served for p = 1, 2 and inf only (got p = %r)" % (p,))
        return _MINKOWSKI[p]
    if metric not in _METRICS and metric not in _SCIPY:
        raise ValueError("metric must be one of %s" % sorted(list(_METRICS) + list(_SCIPY) + ["minkowski"]))
    if p is not None:
        raise ValueError("p is minkowski's order; metric %s takes none" % metric)
    return metric


class SearchResult:
    """recnn/data/db_con.py:5-13: ids int64 [n, topk] and distances fp32 [n, topk], best first."""

    def __init__(self, ids, dist):
        self.ids, self.distances = ids, dist

    def id(self, device=None):
        return self.ids if device is None else self.ids.to(device)

    def dist(self, device=None):
        return self.distances if device is None else self.distances.to(device)


IVF_MAX_DIM = 512          # the fine scan stages a tile of queries and two chunks of list rows in shared memory
IVF_MAX_NPROBE = 64


def ivf_sample(n_items, nlist, seed=0, max_points_per_centroid=256):
    """(sample, init), int64 CPU tensors: the k-means training sample and the positions in it of the initial centroids.
    Every item when n_items <= nlist * max_points_per_centroid, else the first nlist * max_points_per_centroid of
    torch.randperm(n_items) drawn from torch.Generator().manual_seed(seed); init is the first nlist of a second
    randperm(len(sample)) from the same generator."""
    g = torch.Generator().manual_seed(int(seed))
    cap = int(nlist) * int(max_points_per_centroid)
    sample = torch.randperm(n_items, generator=g)[:cap] if n_items > cap else torch.arange(n_items)
    init = torch.randperm(len(sample), generator=g)[:nlist]
    return sample.to(torch.int64), init.to(torch.int64)


PQ_CODEWORDS = 256         # 8-bit codes
PQ_MAX_M = 64
PQ_TRAIN_MAX = 65536       # codebook training points: the first this many of ivf_sample's sample


def ivf_pq_sample(n_sample, seed=0):
    """int64 CPU tensor [256]: the positions, among the first min(n_sample, 65536) points of ivf_sample's sample, of the
    initial codewords of every subspace: the first 256 of torch.randperm(min(n_sample, 65536)) drawn from
    torch.Generator().manual_seed(seed + 1)."""
    n_train = min(int(n_sample), PQ_TRAIN_MAX)
    if n_train < PQ_CODEWORDS:
        raise ValueError("IVF_PQ trains 256 codewords per subspace: it needs a training sample of at least 256 points "
                         "(got %d)" % n_train)
    g = torch.Generator().manual_seed(int(seed) + 1)
    return torch.randperm(n_train, generator=g)[:PQ_CODEWORDS].to(torch.int64)


GRAPH_DEGREES = (16, 32, 64)
GRAPH_MAX_KNN = 64         # the k-NN lists come from a search, whose k is at most 64
GRAPH_MAX_DIM = 512        # a lane of the search keeps at most 16 elements of a row in flight
GRAPH_N_ENTRY = 512        # entry points stored with a graph
GRAPH_KNN_SLAB = 16384     # table rows per k-NN search call


def graph_entry_points(n_items, seed=0):
    """int64 CPU tensor: the first min(512, n_items) ids of torch.randperm(n_items) drawn from
    torch.Generator().manual_seed(seed), the entry points of a graph search (it starts from the first W * degree)"""
    g = torch.Generator().manual_seed(int(seed))
    return torch.randperm(n_items, generator=g)[:GRAPH_N_ENTRY].to(torch.int64)


class IVFLists(NamedTuple):
    """The inverted lists of an ItemIndex: list l holds list_ids[list_offsets[l]:list_offsets[l + 1]], ascending, around
    centroids[l].  The tensors are the index's own device storage: read them, do not write them."""
    centroids: torch.Tensor      # fp32 [nlist, dim]
    list_offsets: torch.Tensor   # int64 [nlist + 1]
    list_ids: torch.Tensor       # int64 [n_items]


class ItemIndex:
    """Exact top-k search over an item-embedding matrix resident on one GPU.

    metric: "L2" (squared Euclidean distance, smallest first -- faiss IndexFlatL2 / Milvus L2),
            "IP" (inner product, largest first), "COS" (cosine similarity, largest first), or a
            scipy.spatial.distance name, smallest first, distances as scipy reports them up to fp32 rounding:
            "euclidean", "cosine" (1 - similarity, clipped to [0, 2]), "cityblock", "chebyshev", "canberra",
            "braycurtis", "correlation", or "minkowski" with ``p`` 1, 2 (the default, as in scipy) or inf, which
            is cityblock, euclidean or chebyshev.  Where scipy gives NaN, Bray-Curtis of two zero rows is 0 and
            correlation with a constant row is 1; a distance that is NaN or +inf (a NaN row, an overflow, Bray-Curtis
            of t = -q != 0) ranks and reports as FLT_MAX.

    ``build_ivf`` turns ``search`` into an IVF_FLAT search (see there); the index is a snapshot of the table at build
    time, which RecNN's workflows keep fixed.  The k-means lists are L2 objects: an index over cityblock, chebyshev,
    canberra, braycurtis or correlation has none.
    """

    def __init__(self, embeddings, metric="L2", p=None):
        name = _metric_name(metric, p)
        if not torch.is_tensor(embeddings):
            embeddings = torch.as_tensor(embeddings)
        if embeddings.device.type != "cuda":
            raise _lib.RecnnError("ItemIndex needs the embedding table on a CUDA device (got %s); there is no CPU path"
                                  % embeddings.device)
        self.table = embeddings.detach().to(torch.float32).contiguous()
        self.metric_name, self.metric = metric, _METRICS.get(name, _SCIPY.get(name))
        self._scipy = name if name in _SCIPY else None
        self.device = self.table.device
        self.n_items, self.dim = int(self.table.shape[0]), int(self.table.shape[1])
        self.norms = None
        if self.metric in (_lib.METRIC_L2, _lib.METRIC_COS, _lib.METRIC_CORR):
            # CORR: the item means, then the centred norms
            n = 2 * self.n_items if self.metric == _lib.METRIC_CORR else self.n_items
            self.norms = torch.empty(n, dtype=torch.float32, device=self.device)
            with torch.cuda.device(self.device):
                _lib.check(_lib.lib().recnn_item_norms(self.table.data_ptr(), self.n_items, self.dim, self.metric,
                                                       self.norms.data_ptr(), _lib.stream_ptr(self.device)))
        self._ws = None
        self._ivf = None
        self._graph = None

    def _result(self, ids, dist):
        """SearchResult, the distances converted for "euclidean" and "cosine"; a -1 pad reports FLT_MAX under every
        scipy name"""
        if self._scipy is not None:
            if self._scipy == "euclidean":
                dist = torch.sqrt(dist)
            elif self._scipy == "cosine":
                dist = torch.clamp(1.0 - dist, 0.0, 2.0)
            dist = torch.where(ids < 0, torch.full_like(dist, _FLT_MAX), dist)
        return SearchResult(ids, dist)

    def _ivf_metric_check(self):
        if self.metric not in _METRICS.values():
            raise ValueError("an IVF index needs metric L2, IP or COS (or euclidean / cosine); its k-means lists do not "
                             "describe %s" % self.metric_name)

    # ------------------------------------------------------------------------------------------------ IVF index
    @property
    def ivf(self):
        """None, or the IVFLists (centroids, list_offsets, list_ids) of the index built by build_ivf / load_ivf."""
        if self._ivf is None:
            return None
        return IVFLists(self._ivf["centroids"], self._ivf["list_offsets"], self._ivf["list_ids"])

    @property
    def pq(self):
        """None, or for an IVF_PQ index (codebooks fp32 [m, 256, dim / m], codes uint8 [n_items, m] in list order: the
        codes of the item list_ids[p] are row p).  Views of the index's own device storage: read them, do not write
        them."""
        if self._ivf is None or "codes" not in self._ivf:
            return None
        return self._ivf["codebooks"], self._ivf["codes"][:, :self._ivf["m"]]

    def _pq_check(self, m):
        m = int(m)
        if not 1 <= m <= PQ_MAX_M or self.dim % m != 0:
            raise ValueError("IVF_PQ needs 1 <= m <= %d dividing dim = %d (got m = %d)" % (PQ_MAX_M, self.dim, m))
        if self.n_items < PQ_CODEWORDS:
            raise ValueError("IVF_PQ trains 256 codewords per subspace: it needs n_items >= 256 (got %d)"
                             % self.n_items)
        return m

    def build_ivf(self, nlist, n_iter=25, seed=0, max_points_per_centroid=256, m=None):
        """Build an inverted-file index over the table on the device and return self: IVF_FLAT when ``m`` is None,
        IVF_PQ with ``m`` one-byte codes per item otherwise.

        k-means (Lloyd, ``n_iter`` rounds) on a sample of at most ``nlist * max_points_per_centroid`` items chosen by
        ``ivf_sample(n_items, nlist, seed, ...)``, initialised at ``nlist`` of its points; empty lists are split as
        faiss does.  COS runs spherical k-means on unit rows, L2 and IP k-means in L2 on the raw rows.  Every item then
        goes to the list of its nearest centroid.  The same table and arguments give the same index, bit for bit.

        IVF_FLAT stores the table a second time, in list order: ``n_items * dim * 4`` bytes, 1 GB at 1M x 256, plus the
        ids and norms.  It is a snapshot of the table at build time.

        IVF_PQ (``m`` dividing dim, 1 <= m <= 64, n_items >= 256) builds the same lists, bit for bit, and stores each item
        as m codes instead of its row: ``n_items * (m + 8)`` bytes plus the centroids and 256 * dim * 4 bytes of
        codebooks (41 MB at 1M x 256, m = 32).  The residual of an item is r = x - c_list(x) (COS: x the unit row);
        subspace j is dims [j * dim / m, (j + 1) * dim / m).  Each subspace's 256 codewords are trained by ``n_iter``
        Lloyd rounds (the coarse build's) on the residuals of the first min(len(sample), 65536) sample points, from the
        codewords ``ivf_pq_sample(len(sample), seed)`` picks; each code is the nearest codeword (fp32, ties to the
        smaller code).  See ``search`` for how the codes are scored."""
        self._ivf_metric_check()
        nlist, n_iter, mppc = int(nlist), int(n_iter), int(max_points_per_centroid)
        if not 1 <= nlist <= self.n_items:
            raise ValueError("nlist must be in [1, n_items = %d] (got %d)" % (self.n_items, nlist))
        if n_iter < 0:
            raise ValueError("n_iter must be >= 0 (got %d)" % n_iter)
        if mppc < 1:
            raise ValueError("max_points_per_centroid must be >= 1 (got %d)" % mppc)
        if self.dim > IVF_MAX_DIM:
            raise ValueError("an IVF index supports dim <= %d (got %d)" % (IVF_MAX_DIM, self.dim))
        if m is not None:
            m = self._pq_check(m)
        sample, init = ivf_sample(self.n_items, nlist, seed, mppc)
        pq_init = ivf_pq_sample(len(sample), seed) if m is not None else None
        dev = self.device
        sample, init = sample.to(dev), init.to(dev)
        ivf = self._ivf_buffers(nlist, m)
        L = _lib.lib()
        with torch.cuda.device(dev):
            if m is None:
                ws = torch.empty(L.recnn_ivf_build_workspace_bytes(self.n_items, self.dim, nlist, len(sample)),
                                 dtype=torch.uint8, device=dev)
                args = _lib.IvfBuildArgs(self._ivf_descriptor(ivf), self.table.data_ptr(), sample.data_ptr(),
                                         len(sample), init.data_ptr(), n_iter, 0, ws.data_ptr(), ws.numel())
                _lib.check(L.recnn_ivf_build(ctypes.byref(args), _lib.stream_ptr(dev)))
            else:
                pq_init = pq_init.to(dev)
                ws = torch.empty(L.recnn_ivf_pq_build_workspace_bytes(self.n_items, self.dim, nlist, len(sample), m),
                                 dtype=torch.uint8, device=dev)
                args = _lib.IvfPqBuildArgs(self._pq_descriptor(ivf), self.table.data_ptr(), sample.data_ptr(),
                                           len(sample), init.data_ptr(), pq_init.data_ptr(), n_iter, 0, ws.data_ptr(),
                                           ws.numel())
                _lib.check(L.recnn_ivf_pq_build(ctypes.byref(args), _lib.stream_ptr(dev)))
        del ws
        ivf["params"] = dict(nlist=nlist, n_iter=n_iter, seed=int(seed), max_points_per_centroid=mppc)
        if m is not None:
            ivf["params"]["m"] = m
        self._ivf_finish(ivf)
        self._graph = None
        return self

    def _ivf_buffers(self, nlist, m=None):
        dev, pitch = self.device, (self.dim + 3) // 4 * 4
        norms = self.metric != _lib.METRIC_IP
        ivf = dict(centroids=torch.empty(nlist, self.dim, dtype=torch.float32, device=dev),
                   centroid_norms=torch.empty(nlist, dtype=torch.float32, device=dev) if norms else None,
                   list_offsets=torch.empty(nlist + 1, dtype=torch.int64, device=dev),
                   list_ids=torch.empty(self.n_items, dtype=torch.int64, device=dev))
        if m is None:
            ivf.update(list_table=torch.empty(self.n_items, pitch, dtype=torch.float32, device=dev),
                       list_norms=torch.empty(self.n_items, dtype=torch.float32, device=dev) if norms else None)
        else:
            # codes rows padded to 16 bytes: the search streams them with bulk copies
            ivf.update(m=m, codebooks=torch.empty(m, PQ_CODEWORDS, self.dim // m, dtype=torch.float32, device=dev),
                       codes=torch.empty(self.n_items, (m + 15) // 16 * 16, dtype=torch.uint8, device=dev))
        return ivf

    def _ivf_descriptor(self, ivf):
        """the recnn_ivf_index of the buffers in ivf"""
        return _lib.ivf_index(self.n_items, self.dim, self.metric, int(ivf["centroids"].shape[0]), ivf["centroids"],
                              ivf["centroid_norms"], ivf["list_offsets"], ivf["list_ids"], ivf["list_table"],
                              ivf["list_norms"])

    def _pq_descriptor(self, ivf):
        """the recnn_ivf_pq_index of the buffers in ivf"""
        return _lib.ivf_pq_index(self.n_items, self.dim, self.metric, int(ivf["centroids"].shape[0]), ivf["m"],
                                 ivf["centroids"], ivf["centroid_norms"], ivf["list_offsets"], ivf["list_ids"],
                                 ivf["codebooks"], ivf["codes"])

    def _ivf_finish(self, ivf):
        ivf["nlist"] = int(ivf["centroids"].shape[0])
        ivf["max_list_len"] = int((ivf["list_offsets"][1:] - ivf["list_offsets"][:-1]).max())
        self._ivf = ivf

    def ivf_state(self):
        """The IVF index as host tensors and plain values, for torch.save: centroids, list_offsets, list_ids, the build
        parameters, the metric and the table's shape; an IVF_PQ index adds its codebooks, and ``m`` to the parameters
        (the codes are rebuilt from the table on loading).  None without an index."""
        if self._ivf is None:
            return None
        state = dict(centroids=self._ivf["centroids"].cpu(), list_offsets=self._ivf["list_offsets"].cpu(),
                     list_ids=self._ivf["list_ids"].cpu(), params=dict(self._ivf["params"]), metric=self.metric_name,
                     n_items=self.n_items, dim=self.dim)
        if "codes" in self._ivf:
            state["codebooks"] = self._ivf["codebooks"].cpu()
        return state

    def load_ivf(self, state):
        """Restore an index saved by ivf_state over this index's table (the same table it was built on) and return
        self.  The shapes and the metric must match, and list_ids must be a permutation of the items, ascending within
        each list, with monotone offsets from 0 to n_items (checked on the device): ValueError otherwise.  The
        list-ordered table and the norms are rebuilt from this index's table.  An IVF_PQ state (``m`` in its params)
        also needs codebooks [m, 256, dim / m]; its codes are encoded again on the device from the table, the lists
        and the codebooks, by the build's kernel, so they equal the build's bit for bit."""
        try:
            cent, offs, ids = state["centroids"], state["list_offsets"], state["list_ids"]
            metric, n_items, dim = state["metric"], int(state["n_items"]), int(state["dim"])
            params = dict(state["params"])
        except (KeyError, TypeError) as e:
            raise ValueError("not an ivf_state() dict: %s" % e)
        self._ivf_metric_check()
        m = params.get("m")
        if m is not None:
            if not isinstance(m, int):
                raise ValueError("malformed ivf state: params['m'] must be an int (got %r)" % (m,))
            m = self._pq_check(m)
            books = state.get("codebooks")
            if (not torch.is_tensor(books) or not books.dtype.is_floating_point
                    or tuple(books.shape) != (m, PQ_CODEWORDS, self.dim // m)):
                raise ValueError("malformed ivf state: an IVF_PQ state needs codebooks [%d, %d, %d] float"
                                 % (m, PQ_CODEWORDS, self.dim // m))
        if metric != self.metric_name:
            raise ValueError("the index was built for metric %s, this ItemIndex is %s" % (metric, self.metric_name))
        if (n_items, dim) != (self.n_items, self.dim):
            raise ValueError("the index was built over a [%d, %d] table, this one is [%d, %d]"
                             % (n_items, dim, self.n_items, self.dim))
        if self.dim > IVF_MAX_DIM:
            raise ValueError("an IVF index supports dim <= %d (got %d)" % (IVF_MAX_DIM, self.dim))
        if not all(torch.is_tensor(t) for t in (cent, offs, ids)):
            raise ValueError("centroids, list_offsets and list_ids must be tensors")
        nlist = int(cent.shape[0]) if cent.dim() == 2 else -1
        if (cent.dim() != 2 or cent.shape[1] != dim or not 1 <= nlist <= n_items or not cent.dtype.is_floating_point
                or tuple(offs.shape) != (nlist + 1,) or tuple(ids.shape) != (n_items,)
                or offs.dtype != torch.int64 or ids.dtype != torch.int64):
            raise ValueError("malformed ivf state: centroids [nlist, %d] float, list_offsets int64 [nlist + 1], "
                             "list_ids int64 [%d]" % (dim, n_items))
        dev = self.device
        offs, ids = offs.to(dev).contiguous(), ids.to(dev).contiguous()
        counts = offs[1:] - offs[:-1]
        ok = bool(offs[0] == 0) and bool(offs[-1] == n_items) and bool((counts >= 0).all())
        if ok:
            ok = bool(((ids >= 0) & (ids < n_items)).all())
        if ok:
            ok = bool((torch.bincount(ids, minlength=n_items) == 1).all())
        if ok and n_items > 1:
            # ascending inside a list: a descent is allowed only where a new list starts
            starts = torch.zeros(n_items, dtype=torch.bool, device=dev)
            starts[offs[1:-1][offs[1:-1] < n_items]] = True
            ok = bool(((ids[1:] > ids[:-1]) | starts[1:]).all())
        if not ok:
            raise ValueError("malformed ivf state: list_ids must be a permutation of [0, %d), ascending within each "
                             "list, and list_offsets monotone from 0 to %d" % (n_items, n_items))
        ivf = self._ivf_buffers(nlist, m)
        ivf["centroids"].copy_(cent.to(device=dev, dtype=torch.float32))
        ivf["list_offsets"].copy_(offs)
        ivf["list_ids"].copy_(ids)
        L = _lib.lib()
        with torch.cuda.device(dev):
            if ivf["centroid_norms"] is not None:
                _lib.check(L.recnn_item_norms(ivf["centroids"].data_ptr(), nlist, self.dim, self.metric,
                                              ivf["centroid_norms"].data_ptr(), _lib.stream_ptr(dev)))
            if m is None:
                _lib.check(L.recnn_ivf_list_table(self.table.data_ptr(), self.n_items, self.dim, self.metric,
                                                  ivf["list_ids"].data_ptr(), ivf["list_table"].data_ptr(),
                                                  _lib.ptr(ivf["list_norms"]), _lib.stream_ptr(dev)))
            else:
                ivf["codebooks"].copy_(books.to(device=dev, dtype=torch.float32))
                ws = torch.empty(L.recnn_ivf_pq_encode_workspace_bytes(self.n_items, self.dim), dtype=torch.uint8,
                                 device=dev)
                args = _lib.IvfPqEncodeArgs(self._pq_descriptor(ivf), self.table.data_ptr(), ws.data_ptr(),
                                            ws.numel())
                _lib.check(L.recnn_ivf_pq_encode(ctypes.byref(args), _lib.stream_ptr(dev)))
                del ws
        ivf["params"] = params
        self._ivf_finish(ivf)
        self._graph = None
        return self

    def _nprobe(self, search_param):
        nlist = self._ivf["nlist"]
        p = dict(search_param or {})
        pq = "codes" in self._ivf
        unknown = sorted(set(p) - ({"nprobe", "refine"} if pq else {"nprobe"}))
        if unknown:
            raise ValueError("unknown search_param keys %s (an %s index takes only %s)"
                             % (unknown, "IVF_PQ" if pq else "IVF_FLAT", "nprobe and refine" if pq else "nprobe"))
        nprobe = int(p.get("nprobe", min(16, nlist)))
        if not 1 <= nprobe <= min(nlist, IVF_MAX_NPROBE):
            raise ValueError("nprobe must be in [1, min(nlist = %d, %d)] (got %d)" % (nlist, IVF_MAX_NPROBE, nprobe))
        return nprobe

    def _refine(self, search_param, topk):
        refine = int((search_param or {}).get("refine", 0))
        if refine < 0 or max(refine, 1) * topk > 64:
            raise ValueError("refine must be >= 0 with refine * topk <= 64 (got refine %d, topk %d)" % (refine, topk))
        return refine

    def search(self, search_vecs, topk=10, search_param=None, exclude=None, exclude_rows=None):
        """search_vecs: [n, dim] (tensor / array on any device).  Returns SearchResult on the index's device.
        ``exclude``: an ``ItemSets`` of item ids never returned (e.g. ``DeviceFrameFeed.seen_items()``), with
        ``exclude_rows`` int64 [n] naming each query's set (-1: none; default query r -> set r).  A query with fewer
        than topk eligible items ends in id -1, distance -FLT_MAX (IP, COS) or FLT_MAX (L2 and every scipy name).  An
        item whose key is NaN or +inf (a NaN row, an overflowing |t|^2, score or distance) ranks as key FLT_MAX: after
        every finite key, ties by id, and before any -1.  An excluded id outside [0, n_items) raises IndexError, a malformed table ValueError.

        Without an IVF index the search is exact and ``search_param`` is ignored.  After ``build_ivf`` / ``load_ivf``
        it is the IVF_FLAT search: ``search_param={"nprobe": p}`` (default 16, at most min(nlist, 64); any other key
        raises ValueError) scans the lists of each query's p nearest centroids, and the result is the exact top-k over
        those lists -- the same for a query whatever other queries share the call.

        On an IVF_PQ index (``build_ivf(..., m=M)``) the probed lists are scored from their codes by asymmetric distance
        computation, in fp32: L2 the squared distance from the query to the item's reconstruction c_list + r_hat (a
        per-(query, list) table of 256 * M entries), IP <q, c_list> + <q, r_hat> (a per-query table), COS the IP form on
        the unit query against the unit-row reconstruction, not renormalised.  ``search_param={"nprobe": p,
        "refine": r}``: r = 0 (default) returns the ADC top-k with ADC distances; r >= 1 re-scores the best r * topk
        ADC candidates exactly against ``table`` (r * topk <= 64) and returns their exact top-k with exact distances,
        computed as IVF_FLAT computes them: when r * topk covers every eligible item of the probed lists, the result is
        IVF_FLAT's at the same nprobe, bit for bit.

        On a graph index (``build_graph`` / ``load_graph``) the search is a beam search over the graph, one CTA per
        query: ``search_param={"itopk_size": T, "search_width": W, "max_iterations": M}`` (Milvus GPU_CAGRA's names;
        defaults 64, 1, 0; T a multiple of 32 in [32, 256] and >= topk, 1 <= W <= 8 with W * graph_degree <= 512,
        M >= 0, 0 meaning until converged; any other key raises ValueError).  A buffer of the T best items found so
        far starts from the first W * graph_degree entry points; each iteration expands the out-lists of the W best
        unexplored entries.  Keys are computed as the flat search computes them (its bits on small-integer tables), and
        a query's result does not depend on the other queries of the call.  Excluded items are traversed but never
        returned: the result is the topk best eligible items of the final buffer, padded as above."""
        from .item_sets import ItemSets, row_map
        nprobe = self._nprobe(search_param) if self._ivf is not None else None
        gparam = self._graph_param(search_param) if self._graph is not None else None
        q = torch.as_tensor(search_vecs)
        if q.dim() == 1:
            q = q.unsqueeze(0)
        if q.dim() != 2 or q.shape[1] != self.dim:
            raise ValueError("search_vecs must be [n, %d]" % self.dim)
        topk = int(topk)
        if not 1 <= topk <= min(64, self.n_items):
            raise ValueError("topk must be in [1, min(64, n_items)]")
        refine = self._refine(search_param, topk) if nprobe is not None and "codes" in self._ivf else None
        if gparam is not None and topk > gparam[0]:
            raise ValueError("topk must be <= itopk_size (got topk %d, itopk_size %d)" % (topk, gparam[0]))
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
        if nprobe is not None:
            return self._ivf_search(q, n, topk, nprobe, sets, rows, refine)
        if gparam is not None:
            return self._graph_search(q, n, topk, gparam, sets, rows)
        need = L.recnn_retrieve_workspace_bytes(n, self.n_items, topk)
        if self._ws is None or self._ws.numel() < need:
            self._ws = torch.empty(need, dtype=torch.uint8, device=self.device)
        args = (q.data_ptr(), n, self.dim, self.table.data_ptr(), self.n_items, _lib.ptr(self.norms), self.metric, topk)
        with torch.cuda.device(self.device):
            if sets is None:
                _lib.check(L.recnn_retrieve_topk(*args, ids.data_ptr(), dist.data_ptr(), self._ws.data_ptr(),
                                                 self._ws.numel(), _lib.stream_ptr(self.device)))
                return self._result(ids, dist)
            sets = sets.to(self.device)
            rows = None if rows is None else rows.to(self.device).contiguous()
            flag = torch.empty(1, dtype=torch.int32, device=self.device)
            _lib.check(L.recnn_retrieve_topk_sets(*args, sets.ids.data_ptr() if sets.ids.numel() else None,
                                                  sets.ids.numel(), sets.offsets.data_ptr(), len(sets),
                                                  _lib.ptr(rows), ids.data_ptr(), dist.data_ptr(), flag.data_ptr(),
                                                  self._ws.data_ptr(), self._ws.numel(),
                                                  _lib.stream_ptr(self.device)))
        self._raise_set_bits(int(flag.item()), len(sets))
        return self._result(ids, dist)

    def _raise_set_bits(self, bits, n_sets):
        if bits & 1:
            raise IndexError("an excluded item id is out of range for the index's %d items" % self.n_items)
        if bits & 4:
            raise ValueError("malformed exclusion table: a set is not ascending, its offsets are out of range or "
                             "decreasing, or an exclude_rows entry is outside [-1, %d)" % n_sets)

    def _ivf_search(self, q, n, topk, nprobe, sets, rows, refine=None):
        L, iv, dev = _lib.lib(), self._ivf, self.device
        ids = torch.empty(n, topk, dtype=torch.int64, device=dev)
        dist = torch.empty(n, topk, dtype=torch.float32, device=dev)
        if refine is None:
            need = L.recnn_ivf_search_workspace_bytes(n, iv["nlist"], nprobe, topk)
        else:
            need = L.recnn_ivf_pq_search_workspace_bytes(n, iv["nlist"], nprobe, topk, refine)
        if self._ws is None or self._ws.numel() < need:
            self._ws = torch.empty(need, dtype=torch.uint8, device=dev)
        set_args, flag = (None, 0, None, 0, None), None
        if sets is not None:
            sets = sets.to(dev)
            rows = None if rows is None else rows.to(dev).contiguous()
            flag = torch.empty(1, dtype=torch.int32, device=dev)
            set_args = (sets.ids.data_ptr() if sets.ids.numel() else None, sets.ids.numel(), sets.offsets.data_ptr(),
                        len(sets), _lib.ptr(rows))
        with torch.cuda.device(dev):
            if refine is None:
                args = _lib.IvfSearchArgs(self._ivf_descriptor(iv), q.data_ptr(), n, nprobe, topk, *set_args,
                                          ids.data_ptr(), dist.data_ptr(), _lib.ptr(flag), self._ws.data_ptr(),
                                          self._ws.numel())
                _lib.check(L.recnn_ivf_search(ctypes.byref(args), _lib.stream_ptr(dev)))
            else:
                args = _lib.IvfPqSearchArgs(self._pq_descriptor(iv), self.table.data_ptr(), _lib.ptr(self.norms),
                                            q.data_ptr(), n, nprobe, topk, refine, 0, *set_args, ids.data_ptr(),
                                            dist.data_ptr(), _lib.ptr(flag), self._ws.data_ptr(), self._ws.numel())
                _lib.check(L.recnn_ivf_pq_search(ctypes.byref(args), _lib.stream_ptr(dev)))
        if flag is not None:
            self._raise_set_bits(int(flag.item()), len(sets))
        return self._result(ids, dist)

    # ---------------------------------------------------------------------------------------------- graph index
    @property
    def graph(self):
        """None, or int32 [n_items, graph_degree]: the out-neighbours of every item in the graph built by build_graph /
        load_graph.  A view of the index's own device storage: read it, do not write it."""
        return None if self._graph is None else self._graph["graph"]

    @property
    def graph_entry(self):
        """None, or int32 [min(512, n_items)]: the entry points of the graph search"""
        return None if self._graph is None else self._graph["entry"]

    def _graph_check(self, d, D):
        self._ivf_metric_check()
        if d not in GRAPH_DEGREES:
            raise ValueError("graph_degree must be one of %s (got %d)" % (GRAPH_DEGREES, d))
        if not d <= D <= GRAPH_MAX_KNN:
            raise ValueError("intermediate_degree must be in [graph_degree = %d, %d]: the k-NN lists come from a search "
                             "whose k is at most %d (got %d)" % (d, GRAPH_MAX_KNN, GRAPH_MAX_KNN, D))
        if self.n_items <= D:
            raise ValueError("a graph index needs n_items > intermediate_degree (got %d items, degree %d)"
                             % (self.n_items, D))
        if self.dim > GRAPH_MAX_DIM:
            raise ValueError("a graph index supports dim <= %d (got %d)" % (GRAPH_MAX_DIM, self.dim))

    def knn_lists(self, degree, knn_nlist=None, knn_nprobe=None):
        """int64 [n_items, degree] on the index's device: row u holds u's ``degree`` best items by (key, id) under the
        index's metric, u itself excluded through an ItemSets of one id per row.  Exact (the flat search, in slabs of
        16,384 rows) by default; with ``knn_nlist`` from an IVF_FLAT index of that many lists, built for the purpose
        and freed after, probed at ``knn_nprobe`` (default min(16, knn_nlist)); a row whose probed lists hold fewer
        than ``degree`` eligible items is searched again exactly."""
        from .item_sets import ItemSets
        n, dev = self.n_items, self.device
        flat = ItemIndex(self.table, self.metric_name)
        selves = ItemSets(torch.arange(n, device=dev), torch.arange(n + 1, device=dev))
        approx, param = flat, None
        if knn_nlist is not None:
            approx = ItemIndex(self.table, self.metric_name).build_ivf(int(knn_nlist))
            param = {"nprobe": int(knn_nprobe) if knn_nprobe is not None else min(16, int(knn_nlist))}
        elif knn_nprobe is not None:
            raise ValueError("knn_nprobe needs knn_nlist")
        out = torch.empty(n, degree, dtype=torch.int64, device=dev)
        for r0 in range(0, n, GRAPH_KNN_SLAB):
            rows = torch.arange(r0, min(n, r0 + GRAPH_KNN_SLAB), device=dev)
            out[r0:r0 + len(rows)] = approx.search(self.table[rows], degree, search_param=param, exclude=selves,
                                                   exclude_rows=rows).ids
        del approx
        if knn_nlist is not None:
            short = (out < 0).any(1).nonzero().flatten()
            for s0 in range(0, len(short), GRAPH_KNN_SLAB):
                rows = short[s0:s0 + GRAPH_KNN_SLAB]
                out[rows] = flat.search(self.table[rows], degree, exclude=selves, exclude_rows=rows).ids
        return out

    def build_graph(self, graph_degree=32, intermediate_degree=64, knn_nlist=None, knn_nprobe=None, seed=0):
        """Build a proximity-graph index over the table on the device (CAGRA's construction) and return self; it
        replaces an IVF index.  Metric L2, IP or COS (or euclidean / cosine), graph_degree d in {16, 32, 64},
        d <= intermediate_degree D <= 64 < n_items, dim <= 512.

        1. k-NN lists: N(u) = u's D best items (``knn_lists``: exact, or through a temporary IVF_FLAT index with
           ``knn_nlist`` / ``knn_nprobe``).
        2. Pruning: c_j = the number of i < j such that v_j is in N(v_i) at a position p < j; P(u) keeps the d
           positions first in (c_j, j) order.
        3. Reverse edges: each kept edge u -> v at rank r makes u a reverse candidate of v, ordered by (r, u).
        4. Merge: v's out-list is the first d/2 of P(v), then its reverse candidates, then the rest of P(v), skipping
           repeats, until it holds d ids: every item gets d distinct out-neighbours and no self-loop.
        5. Entry points: ``graph_entry_points(n_items, seed)``.

        Steps 2-4 run on the device (recnn_graph_build) on integer data only, so the graph is a function of the k-NN
        ids, bit for bit.  The index holds n_items * d int32 ids (128 MB at 1M items, d = 32) and reads the table
        itself: it is a snapshot of the table at build time."""
        d, D = int(graph_degree), int(intermediate_degree)
        self._graph_check(d, D)
        knn = self.knn_lists(D, knn_nlist, knn_nprobe)
        gr = self._graph_buffers(d, graph_entry_points(self.n_items, seed))
        L, dev = _lib.lib(), self.device
        flag = torch.zeros(1, dtype=torch.int32, device=dev)
        with torch.cuda.device(dev):
            ws = torch.empty(L.recnn_graph_build_workspace_bytes(self.n_items, d), dtype=torch.uint8, device=dev)
            args = _lib.GraphBuildArgs(self._graph_descriptor(gr), knn.data_ptr(), D, 0, flag.data_ptr(),
                                       ws.data_ptr(), ws.numel())
            _lib.check(L.recnn_graph_build(ctypes.byref(args), _lib.stream_ptr(dev)))
        del ws, knn
        if int(flag.item()) != 0:
            raise _lib.RecnnError("the k-NN lists of the graph build were malformed (error bits %d)" % int(flag.item()))
        gr["params"] = dict(graph_degree=d, intermediate_degree=D, knn_nlist=knn_nlist, knn_nprobe=knn_nprobe,
                            seed=int(seed))
        self._graph, self._ivf = gr, None
        return self

    def _graph_buffers(self, d, entry):
        dev = self.device
        return dict(graph=torch.empty(self.n_items, d, dtype=torch.int32, device=dev),
                    entry=entry.to(device=dev, dtype=torch.int32).contiguous(), degree=d)

    def _graph_descriptor(self, gr):
        """the recnn_graph_index of the buffers in gr"""
        return _lib.graph_index(self.n_items, self.dim, self.metric, gr["degree"], self.table, self.norms,
                                gr["graph"], gr["entry"])

    def graph_state(self):
        """The graph index as host tensors and plain values, for torch.save: graph int32 [n_items, d], entry int32,
        the build parameters, the metric and the table's shape.  None without a graph."""
        if self._graph is None:
            return None
        return dict(graph=self._graph["graph"].cpu(), entry=self._graph["entry"].cpu(),
                    params=dict(self._graph["params"]), metric=self.metric_name, n_items=self.n_items, dim=self.dim)

    def load_graph(self, state):
        """Restore a graph saved by graph_state over this index's table (the one it was built on) and return self; it
        replaces an IVF index.  The metric and shapes must match, every id must be in [0, n_items), and no graph row
        may hold its own item or a repeated id (checked on the device): ValueError otherwise."""
        try:
            graph, entry = state["graph"], state["entry"]
            metric, n_items, dim = state["metric"], int(state["n_items"]), int(state["dim"])
            params = dict(state["params"])
        except (KeyError, TypeError) as e:
            raise ValueError("not a graph_state() dict: %s" % e)
        self._ivf_metric_check()
        if metric != self.metric_name:
            raise ValueError("the graph was built for metric %s, this ItemIndex is %s" % (metric, self.metric_name))
        if (n_items, dim) != (self.n_items, self.dim):
            raise ValueError("the graph was built over a [%d, %d] table, this one is [%d, %d]"
                             % (n_items, dim, self.n_items, self.dim))
        if self.dim > GRAPH_MAX_DIM:
            raise ValueError("a graph index supports dim <= %d (got %d)" % (GRAPH_MAX_DIM, self.dim))
        if not (torch.is_tensor(graph) and torch.is_tensor(entry)):
            raise ValueError("graph and entry must be tensors")
        n_entry = min(GRAPH_N_ENTRY, n_items)
        if (graph.dim() != 2 or graph.shape[0] != n_items or int(graph.shape[1]) not in GRAPH_DEGREES
                or int(graph.shape[1]) >= n_items or graph.dtype != torch.int32
                or tuple(entry.shape) != (n_entry,) or entry.dtype != torch.int32):
            raise ValueError("malformed graph state: graph int32 [%d, d] with d in %s, entry int32 [%d]"
                             % (n_items, GRAPH_DEGREES, n_entry))
        dev = self.device
        g, e = graph.to(dev).contiguous(), entry.to(dev).contiguous()
        ok = bool(((g >= 0) & (g < n_items)).all()) and bool(((e >= 0) & (e < n_items)).all())
        if ok:
            srt = torch.sort(g, dim=1).values
            self_loop = (g == torch.arange(n_items, device=dev, dtype=torch.int32)[:, None]).any()
            ok = not bool(self_loop) and not bool((srt[:, 1:] == srt[:, :-1]).any())
        if ok:
            se = torch.sort(e).values
            ok = not bool((se[1:] == se[:-1]).any())
        if not ok:
            raise ValueError("malformed graph state: every id must be in [0, %d), no graph row may hold its own item "
                             "or a repeated id, and the entry points must be distinct" % n_items)
        gr = self._graph_buffers(int(graph.shape[1]), e)
        gr["graph"].copy_(g)
        gr["params"] = params
        self._graph, self._ivf = gr, None
        return self

    def _graph_param(self, search_param):
        p = dict(search_param or {})
        unknown = sorted(set(p) - {"itopk_size", "search_width", "max_iterations"})
        if unknown:
            raise ValueError("unknown search_param keys %s (a graph index takes only itopk_size, search_width and "
                             "max_iterations)" % unknown)
        T, W, M = int(p.get("itopk_size", 64)), int(p.get("search_width", 1)), int(p.get("max_iterations", 0))
        d = self._graph["degree"]
        if not (32 <= T <= 256 and T % 32 == 0):
            raise ValueError("itopk_size must be a multiple of 32 in [32, 256] (got %d)" % T)
        if not (1 <= W <= 8 and W * d <= 512):
            raise ValueError("search_width must be in [1, 8] with search_width * graph_degree <= 512 (got %d, degree "
                             "%d)" % (W, d))
        if M < 0:
            raise ValueError("max_iterations must be >= 0 (got %d)" % M)
        return T, W, M

    def _graph_search(self, q, n, topk, gparam, sets, rows, iterations=None):
        L, gr, dev = _lib.lib(), self._graph, self.device
        T, W, M = gparam
        ids = torch.empty(n, topk, dtype=torch.int64, device=dev)
        dist = torch.empty(n, topk, dtype=torch.float32, device=dev)
        need = L.recnn_graph_search_workspace_bytes(n, T)
        if self._ws is None or self._ws.numel() < need:
            self._ws = torch.empty(need, dtype=torch.uint8, device=dev)
        set_args, flag = (None, 0, None, 0, None), None
        if sets is not None:
            sets = sets.to(dev)
            rows = None if rows is None else rows.to(dev).contiguous()
            flag = torch.empty(1, dtype=torch.int32, device=dev)
            set_args = (sets.ids.data_ptr() if sets.ids.numel() else None, sets.ids.numel(), sets.offsets.data_ptr(),
                        len(sets), _lib.ptr(rows))
        with torch.cuda.device(dev):
            args = _lib.GraphSearchArgs(self._graph_descriptor(gr), q.data_ptr(), n, topk, T, W, M, *set_args,
                                        ids.data_ptr(), dist.data_ptr(), _lib.ptr(iterations), _lib.ptr(flag),
                                        self._ws.data_ptr(), self._ws.numel())
            _lib.check(L.recnn_graph_search(ctypes.byref(args), _lib.stream_ptr(dev)))
        if flag is not None:
            self._raise_set_bits(int(flag.item()), len(sets))
        return self._result(ids, dist)

    def graph_iterations(self, search_vecs, search_param=None):
        """int32 [n]: the iterations past the entry step that ``search`` runs for each query at these parameters (the
        same for every topk), e.g. to see how long a search takes to converge"""
        if self._graph is None:
            raise ValueError("graph_iterations needs a graph index (build_graph / load_graph)")
        T, W, M = self._graph_param(search_param)
        q = torch.as_tensor(search_vecs)
        if q.dim() == 1:
            q = q.unsqueeze(0)
        if q.dim() != 2 or q.shape[1] != self.dim:
            raise ValueError("search_vecs must be [n, %d]" % self.dim)
        q = q.detach().to(device=self.device, dtype=torch.float32).contiguous()
        it = torch.zeros(q.shape[0], dtype=torch.int32, device=self.device)
        if q.shape[0]:
            self._graph_search(q, int(q.shape[0]), 1, (T, W, M), None, None, iterations=it)
        return it

    def rank(self, search_vecs, target, exclude=None, exclude_rows=None):
        """int64 [n]: for offline evaluation, the number of items ``search`` on the same queries would return before
        ``target[q]`` (better key, equal keys the smaller id), i.e. the target's position in ``search(vecs, k)`` when
        below k and the target is absent otherwise, at any k.  Ranks are always the exact ones, also on an index with
        IVF lists, so the recall of an ``nprobe`` can be measured against them.  ``exclude`` / ``exclude_rows`` as in ``search``; a
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
    is ``env.base.embeddings``; ``param["metric_type"]`` may be "L2" (default) or "IP".  ``param["index_type"]``
    "IVF_FLAT" with ``param["nlist"]`` builds the IVF index at construction (Milvus create_index(IVF_FLAT, {"nlist"})),
    so that ``search(..., search_param={"nprobe": p})`` means what it means to Milvus; "IVF_PQ" with ``param["nlist"]``,
    ``param["m"]`` and optionally ``param["nbits"]`` (8, the only width) builds the IVF_PQ index (Milvus
    create_index(IVF_PQ, {"nlist", "m", "nbits"})); "GPU_CAGRA" with optional ``param["intermediate_graph_degree"]``
    (default 64) and ``param["graph_degree"]`` (default 32, both at most 64) builds the graph index (build_graph), searched
    with search_param {"itopk_size", "search_width", "max_iterations"}; without it, or with "FLAT", the search is exact.
    No Milvus server is involved."""

    def __init__(self, env, name="movies_L2", port="19530", param=None):
        metric = "L2"
        if param and "metric_type" in param:
            mt = str(param["metric_type"]).upper()
            metric = "IP" if mt.endswith("IP") else "L2"
        index_type = str(param.get("index_type", "FLAT")).upper() if param else "FLAT"
        if index_type not in ("FLAT", "IVF_FLAT", "IVF_PQ", "GPU_CAGRA"):
            raise ValueError("index_type must be FLAT, IVF_FLAT, IVF_PQ or GPU_CAGRA (got %s)" % index_type)
        if index_type in ("IVF_FLAT", "IVF_PQ") and "nlist" not in param:
            raise ValueError("index_type %s needs param['nlist']" % index_type)
        if index_type == "IVF_PQ":
            if "m" not in param:
                raise ValueError("index_type IVF_PQ needs param['m']")
            if int(param.get("nbits", 8)) != 8:
                raise ValueError("IVF_PQ supports nbits = 8 only (got %s)" % param["nbits"])
        if index_type == "GPU_CAGRA":
            D, d = int(param.get("intermediate_graph_degree", 64)), int(param.get("graph_degree", 32))
            if D > GRAPH_MAX_KNN or d > GRAPH_MAX_KNN:
                raise ValueError("GPU_CAGRA supports intermediate_graph_degree and graph_degree up to %d (got %d, %d): "
                                 "the k-NN lists are built by the search, whose k is at most %d"
                                 % (GRAPH_MAX_KNN, D, d, GRAPH_MAX_KNN))
        emb = env.base.embeddings if hasattr(env, "base") else env
        super().__init__(emb, metric)
        if index_type == "GPU_CAGRA":
            self.build_graph(graph_degree=d, intermediate_degree=D)
        elif index_type == "IVF_FLAT":
            self.build_ivf(int(param["nlist"]))
        elif index_type == "IVF_PQ":
            self.build_ivf(int(param["nlist"]), m=int(param["m"]))
        self.name = name
        self.statuses = {}

    def get_log(self):
        return self.statuses
