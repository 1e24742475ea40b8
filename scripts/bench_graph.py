"""Graph-index search (ItemIndex.build_graph + search(..., search_param={"itopk_size": T, "search_width": W})) against
the flat search and IVF_FLAT in the same process.

Prints one JSON line.  Tables (bench_ivf.py's generators): 1,000,000 x 256 "mixture" and "iid", and the ML-20M shape
26,744 x 128 "mixture".  Build (graph_degree 32, intermediate_degree 64): one call each with the exact k-NN lists and
with IVF k-NN lists (knn_nlist 1,024, knn_nprobe 16), CUDA-event time, the bytes the index holds, and the recall@10
of each graph at T 64, W 1.  Search over the exact-k-NN graph: median / min / max CUDA-event time of --repeats calls
after --warmup, for 1 / 128 / 2,048 / 16,384 queries, k 10, T 32 / 64 / 128 / 256, W 1 / 4, recall@10 against the
flat ids and the mean iterations to convergence; the flat search and IVF_FLAT (nlist 1,024, nprobe 1 / 4 / 16) of
the same queries alongside.  Cost model (a model figure, not a measurement): a query reads at most
(iterations + 1) * W * graph_degree rows of dim * 4 bytes (repeats are dropped before reading, so fewer in fact); that
many bytes over the kernel time, as a share of the H100 SXM data sheet's 3.35 TB/s.  The card's name, power limit and
maximum SM clock are read in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "scripts")):
    if p not in sys.path:
        sys.path.insert(0, p)

from recnn_b200.data import ItemIndex  # noqa: E402
from recnn_b200.utils.metrics import recall_at_k  # noqa: E402
from bench_recommend import gpu_info, timed  # noqa: E402
from bench_ivf import make_queries, make_table  # noqa: E402

TABLES = (("mixture", 1_000_000, 256), ("iid", 1_000_000, 256), ("mixture", 26_744, 128))
QUERIES, K = (1, 128, 2048, 16384), 10
ITOPK, WIDTHS, NPROBES = (32, 64, 128, 256), (1, 4), (1, 4, 16)
DEGREE, KNN_DEGREE, KNN_NLIST, KNN_NPROBE, NLIST = 32, 64, 1024, 16, 1024
HBM = 3.35e12


def event_time(fn):
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    torch.cuda.synchronize()
    ev[0].record()
    out = fn()
    ev[1].record()
    ev[1].synchronize()
    return ev[0].elapsed_time(ev[1]) / 1e3, out


def graph_bytes(index):
    return index.graph.numel() * 4 + index.graph_entry.numel() * 4


def table_case(kind, items, dim, warmup, repeats, ivf_knn):
    table, g = make_table(kind, items, dim, items + dim)
    flat = ItemIndex(table, "L2")
    out = {"table": kind, "items": items, "dim": dim, "build": []}
    probe_q = make_queries(kind, table, 2048, g)
    probe_exact = flat.search(probe_q, K).ids
    builds = [("exact", {})] + ([("ivf", {"knn_nlist": KNN_NLIST, "knn_nprobe": KNN_NPROBE})] if ivf_knn else [])
    index = None
    for name, kw in builds:
        t, idx = event_time(lambda: ItemIndex(table, "L2").build_graph(DEGREE, KNN_DEGREE, **kw))
        rec = recall_at_k(idx.search(probe_q, K, search_param={"itopk_size": 64}).ids, probe_exact)[1]
        out["build"].append({"knn": name, **kw, "time_s": t, "index_bytes": graph_bytes(idx),
                             "recall10_T64_W1_2048q": rec})
        if index is None:
            index = idx
        else:
            del idx
    t, ivf = event_time(lambda: ItemIndex(table, "L2").build_ivf(NLIST))
    out["ivf_flat"] = {"nlist": NLIST, "build_time_s": t,
                       "index_bytes": sum(v.numel() * v.element_size() for v in ivf._ivf.values() if torch.is_tensor(v))}
    out["search"] = []
    for n in QUERIES:
        q = make_queries(kind, table, n, g)
        exact = flat.search(q, K).ids
        res = {"queries": n, "k": K, "flat": timed(lambda: flat.search(q, K), warmup, repeats), "ivf_flat": [],
               "graph": []}
        for p in NPROBES:
            prm = {"nprobe": p}
            res["ivf_flat"].append({"nprobe": p, "time": timed(lambda: ivf.search(q, K, search_param=prm), warmup,
                                                              repeats),
                                    "recall": recall_at_k(ivf.search(q, K, search_param=prm).ids, exact)[1]})
        for T in ITOPK:
            for W in WIDTHS:
                prm = {"itopk_size": T, "search_width": W}
                r = {"itopk_size": T, "search_width": W,
                     "time": timed(lambda: index.search(q, K, search_param=prm), warmup, repeats),
                     "recall": recall_at_k(index.search(q, K, search_param=prm).ids, exact)[1]}
                it = index.graph_iterations(q, prm).double()
                r["iterations_mean"] = float(it.mean())
                r["iterations_max"] = int(it.max())
                rows = float(((it + 1) * W * DEGREE).sum())
                nbytes = rows * dim * 4
                r["model_rows_per_query"] = rows / n
                r["model_share_of_hbm"] = nbytes / HBM / r["time"]["time_s_median"]
                res["graph"].append(r)
        out["search"].append(res)
    del ivf, index, flat, table
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--tables", default="0,1,2", help="indices into TABLES")
    ap.add_argument("--no-ivf-knn", action="store_true", help="skip the IVF k-NN build")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_graph.py needs a GPU")
    result = {"metric": "graph", **gpu_info(), "cases": []}
    for ti in (int(x) for x in args.tables.split(",")):
        kind, items, dim = TABLES[ti]
        result["cases"].append(table_case(kind, items, dim, args.warmup, args.repeats, not args.no_ivf_knn))
        print(json.dumps(result["cases"][-1]), file=sys.stderr, flush=True)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
