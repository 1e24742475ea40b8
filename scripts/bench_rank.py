"""Offline evaluation: the exact rank of each row's held-out item (DiscreteActor.rank, ItemIndex.rank) against the
serving call it is defined by (DiscreteActor.topk at k 10, ItemIndex.search at k 10).

Prints one JSON line.  The policy (S 2570 / H 256 / 1,000,000 items, rows 128, 2,048 and 16,384) runs rank and topk
without exclusion and with a whole-history ItemSets table per row (the long-tailed histories of bench_recommend.py).
Retrieval (L2, 128 and 2,048 queries) runs over a 26,744 x 128 table and a 1,000,000 x 256 one, without and with
history sets.  Targets are uniform item ids.

Per case: the median / min / max CUDA-event time of one call over --repeats calls after --warmup calls and the peak
torch.cuda.max_memory_allocated() above the inputs during one call, as bench_recommend.py measures them; each rank case
carries its time ratio to the serving call on the same inputs.  The card's name, power limit and maximum SM clock are
read in the same run.
"""
from __future__ import annotations

import argparse
import gc
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "scripts")):
    if p not in sys.path:
        sys.path.insert(0, p)

import recnn_b200  # noqa: E402
from recnn_b200.nn.arena import param_arena  # noqa: E402
from bench_recommend import gpu_info, histories, timed  # noqa: E402

S, H, ITEMS = 2570, 256, 1_000_000
ROWS = (128, 2048, 16384)
K = 10
TABLES = ((26_744, 128), (1_000_000, 256))
QUERIES = (128, 2048)


def ratio(res, rank, serve):
    res[rank]["time_ratio_to_" + serve] = res[rank]["time_s_median"] / res[serve]["time_s_median"]


def policy_cases(warmup, repeats):
    torch.manual_seed(1)
    with torch.device("cuda"):
        m = recnn_b200.nn.DiscreteActor(S, ITEMS, H)
    param_arena(m)
    out = []
    for N in ROWS:
        g = torch.Generator(device="cuda").manual_seed(N)
        state = torch.randn(N, S, device="cuda", generator=g)
        target = torch.randint(0, ITEMS, (N,), device="cuda", generator=g)
        sets, lengths = histories(N, ITEMS, N)
        res = {"rows": N, "k": K, "num_items": ITEMS, "mean_set": float(lengths.mean()), "max_set": int(lengths.max())}
        res["topk_none"] = timed(lambda: m.topk(state, K), warmup, repeats)
        res["rank_none"] = timed(lambda: m.rank(state, target), warmup, repeats)
        res["topk_sets"] = timed(lambda: m.topk(state, K, exclude=sets), warmup, repeats)
        res["rank_sets"] = timed(lambda: m.rank(state, target, exclude=sets), warmup, repeats)
        ratio(res, "rank_none", "topk_none")
        ratio(res, "rank_sets", "topk_sets")
        out.append(res)
        del state, target, sets
        gc.collect()
        torch.cuda.empty_cache()
    del m
    gc.collect()
    torch.cuda.empty_cache()
    return out


def retrieval_cases(warmup, repeats):
    from recnn_b200.data import ItemIndex
    out = []
    for items, dim in TABLES:
        g = torch.Generator(device="cuda").manual_seed(items)
        table = torch.randn(items, dim, device="cuda", generator=g)
        index = ItemIndex(table, "L2")
        for n in QUERIES:
            q = torch.randn(n, dim, device="cuda", generator=g)
            target = torch.randint(0, items, (n,), device="cuda", generator=g)
            sets, lengths = histories(n, items, n + 1)
            res = {"items": items, "dim": dim, "queries": n, "k": K, "metric": "L2",
                   "mean_set": float(lengths.mean()), "max_set": int(lengths.max())}
            res["search_none"] = timed(lambda: index.search(q, K), warmup, repeats)
            res["rank_none"] = timed(lambda: index.rank(q, target), warmup, repeats)
            res["search_sets"] = timed(lambda: index.search(q, K, exclude=sets), warmup, repeats)
            res["rank_sets"] = timed(lambda: index.rank(q, target, exclude=sets), warmup, repeats)
            ratio(res, "rank_none", "search_none")
            ratio(res, "rank_sets", "search_sets")
            out.append(res)
        del index, table
        gc.collect()
        torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--repeats", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_rank.py needs a GPU")
    result = {"metric": "rank", **gpu_info(), "S": S, "H": H}
    result["policy"] = policy_cases(args.warmup, args.repeats)
    result["retrieval"] = retrieval_cases(args.warmup, args.repeats)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
