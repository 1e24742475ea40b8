"""IVF_FLAT search (ItemIndex.build_ivf + search(..., search_param={"nprobe": p})) against the exact flat search.

Prints one JSON line.  Tables: the ML-20M shape (26,744 x 128) and 1,000,000 x 256, each built two ways:
  - "mixture": a seeded Gaussian mixture (4,096 components, N(0, 1) centres, per-dimension spread 0.25; queries are
    items plus the same noise), the clustered structure real item embeddings have and IVF exploits;
  - "iid": N(0, 1) rows, IVF's worst case: no structure, so each list is a Voronoi cell of noise and recall per probed
    list is lowest.
Build: time (one call, CUDA events) and index bytes at nlist 1,024 and 4,096.  Search (nlist 1,024): median / min / max
CUDA-event time over --repeats calls after --warmup, at 128 / 2,048 / 16,384 queries x k 10 / 64 x nprobe 1 / 4 / 16 / 64,
with the flat search of the same queries alongside, and recall@k (recnn_b200.utils.metrics.recall_at_k) against the
flat ids; with the long-tailed history sets of bench_recommend.py at nprobe 16.  Cost model of the fine scan: each
work unit (a list and up to 32 of the queries probing it) reads its list's rows once, so bytes = sum over units of
list length x pitch x 4, FLOPs = 2 x dim x the (query, item) pairs scanned; the least time the H100 SXM data sheet
allows (3.35 TB/s, 67 TFLOP/s dense FP32 for a card allowed 700 W) and which of the two bounds it.  Wolpertinger
candidate step at 2,048 rows over the 1M table: actor + IVF search(64) against actor + flat search(64), then
Critic.topk(10) over the 64 candidates.  The card's name, power limit and maximum SM clock are read in the same run.
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

import recnn_b200  # noqa: E402
from recnn_b200.data import ItemIndex  # noqa: E402
from recnn_b200.nn.arena import param_arena  # noqa: E402
from recnn_b200.utils.metrics import recall_at_k  # noqa: E402
from bench_recommend import gpu_info, histories, timed  # noqa: E402

TABLES = ((26_744, 128), (1_000_000, 256))
QUERIES, KS, NPROBES = (128, 2048, 16384), (10, 64), (1, 4, 16, 64)
NLISTS = (1024, 4096)
HBM = 3.35e12
FP32 = 67e12
SPREAD = 0.25                # per-dimension spread of a mixture component around its N(0, 1) centre


def make_table(kind, items, dim, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    if kind == "iid":
        return torch.randn(items, dim, device="cuda", generator=g), g
    centres = torch.randn(4096, dim, device="cuda", generator=g)
    comp = torch.randint(0, 4096, (items,), device="cuda", generator=g)
    return centres[comp] + SPREAD * torch.randn(items, dim, device="cuda", generator=g), g


def make_queries(kind, table, n, g):
    """queries near items (an item plus noise): what an actor's action looks like against a clustered table"""
    if kind == "iid":
        return torch.randn(n, table.shape[1], device="cuda", generator=g)
    pick = torch.randint(0, table.shape[0], (n,), device="cuda", generator=g)
    return table[pick] + SPREAD * torch.randn(n, table.shape[1], device="cuda", generator=g)


def index_bytes(index):
    return sum(t.numel() * t.element_size() for t in index._ivf.values() if torch.is_tensor(t))


def fine_scan_cost(index, q, nprobe):
    iv = index._ivf
    probes = ItemIndex(iv["centroids"], index.metric_name).search(q, nprobe).ids.reshape(-1)
    cnt = torch.bincount(probes, minlength=iv["nlist"]).double()
    lens = (iv["list_offsets"][1:] - iv["list_offsets"][:-1]).double()
    pitch = iv["list_table"].shape[1]
    units = torch.ceil(cnt / 32)
    nbytes = float((units * lens).sum()) * pitch * 4
    flops = 2.0 * index.dim * float((cnt * lens).sum())
    return nbytes, flops


def table_cases(kind, items, dim, warmup, repeats):
    table, g = make_table(kind, items, dim, items + dim)
    flat = ItemIndex(table, "L2")
    out = {"table": kind, "items": items, "dim": dim, "build": [], "search": []}
    index = None
    for nlist in NLISTS:
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        torch.cuda.synchronize()
        ev[0].record()
        idx = ItemIndex(table, "L2").build_ivf(nlist)
        ev[1].record()
        ev[1].synchronize()
        out["build"].append({"nlist": nlist, "time_s": ev[0].elapsed_time(ev[1]) / 1e3, "index_bytes": index_bytes(idx),
                             "max_list_len": idx._ivf["max_list_len"]})
        if nlist == 1024:
            index = idx
        else:
            del idx
    for n in QUERIES:
        q = make_queries(kind, table, n, g)
        sets = histories(n, items, n)[0] if n <= 2048 else None
        for k in KS:
            exact = flat.search(q, k).ids
            res = {"queries": n, "k": k, "flat": timed(lambda: flat.search(q, k), warmup, repeats), "ivf": []}
            for p in NPROBES:
                r = {"nprobe": p, "time": timed(lambda: index.search(q, k, search_param={"nprobe": p}), warmup,
                                                repeats)}
                r["recall"] = recall_at_k(index.search(q, k, search_param={"nprobe": p}).ids, exact)[1]
                nbytes, flops = fine_scan_cost(index, q, p)
                t = r["time"]["time_s_median"]
                r.update(fine_scan_bytes=nbytes, fine_scan_flops=flops,
                         bound="hbm" if nbytes / HBM > flops / FP32 else "fp32",
                         share_of_bound=max(nbytes / HBM, flops / FP32) / t)
                if p == 16 and sets is not None:
                    r["with_sets"] = timed(lambda: index.search(q, k, search_param={"nprobe": p}, exclude=sets),
                                           warmup, repeats)
                    r["flat_with_sets"] = timed(lambda: flat.search(q, k, exclude=sets), warmup, repeats)
                res["ivf"].append(r)
            out["search"].append(res)
    return out, table, index, flat


def wolpertinger(table, index, flat, warmup, repeats):
    S, A, H, N = 2570, table.shape[1], 256, 2048
    torch.manual_seed(1)
    with torch.device("cuda"):
        critic = recnn_b200.nn.Critic(S, A, H).eval()
        actor = recnn_b200.nn.Actor(S, A, H).eval()
    param_arena(critic)
    param_arena(actor)
    state = torch.randn(N, S, device="cuda", generator=torch.Generator(device="cuda").manual_seed(2))
    res = {"rows": N, "S": S, "A": A, "H": H, "nlist": index._ivf["nlist"]}
    res["actor_flat_search64"] = timed(lambda: flat.search(actor(state), 64), warmup, repeats)
    exact = flat.search(actor(state), 64).ids
    for p in (4, 16):
        res["actor_ivf_search64_nprobe%d" % p] = timed(
            lambda: index.search(actor(state), 64, search_param={"nprobe": p}), warmup, repeats)
        res["recall64_nprobe%d" % p] = recall_at_k(index.search(actor(state), 64, search_param={"nprobe": p}).ids,
                                                   exact)[1]
    cand = index.search(actor(state), 64, search_param={"nprobe": 16}).id()
    res["critic_topk10_over_64"] = timed(lambda: critic.topk(state, 10, table, candidates=cand), warmup, repeats)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--tables", default="0,1", help="indices into TABLES")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_ivf.py needs a GPU")
    result = {"metric": "ivf", **gpu_info(), "cases": []}
    for ti in (int(x) for x in args.tables.split(",")):
        items, dim = TABLES[ti]
        for kind in ("mixture", "iid"):
            out, table, index, flat = table_cases(kind, items, dim, args.warmup, args.repeats)
            if items == 1_000_000 and kind == "mixture":
                out["wolpertinger"] = wolpertinger(table, index, flat, args.warmup, args.repeats)
            result["cases"].append(out)
            del table, index, flat
            torch.cuda.empty_cache()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
