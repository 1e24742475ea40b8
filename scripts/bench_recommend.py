"""Serving recommendations that skip what a user has already rated: DiscreteActor.topk and ItemIndex.search with and
without exclusion sets.

Prints one JSON line.  The policy (S 2570 / H 256 / 1,000,000 items, rows 1, 128, 2,048 and 16,384, k 10 and 64) runs
three ways: no exclusion, the frame's 10 ids as a dense [N, 10] list (recnn_discrete_topk), and a whole-history
ItemSets table per row (recnn_discrete_topk_sets).  Retrieval (ItemIndex.search, L2, k 10, 128 and 2,048 queries) runs
over a 26,744 x 128 table (the ML-20M item count) and a 1,000,000 x 256 one, without and with history sets.  The
histories are fixed-seed, long-tailed (Lomax lengths, mean about 144 -- ML-20M's 20,000,263 ratings over 138,493 users
-- with every 256th row at 8,192 or more) and hold uniformly drawn ids.

Per case: the median / min / max CUDA-event time of one call over --repeats calls after --warmup calls, and the peak
torch.cuda.max_memory_allocated() above the inputs during one call (workspace included; the set table is an input).
The time ratio of each exclusion case to the same shape without exclusion is reported beside it.  The card's name,
power limit and maximum SM clock are read in the same run.

``--cases`` picks a subset (e.g. ``policy_none,policy_frame`` to time the calls that existed before sets).
"""
from __future__ import annotations

import argparse
import gc
import json
import os
import statistics
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import recnn_b200  # noqa: E402
from recnn_b200.nn.arena import param_arena  # noqa: E402

S, H, ITEMS = 2570, 256, 1_000_000
ROWS = (1, 128, 2048, 16384)
KS = (10, 64)
FRAME = 10
TABLES = ((26_744, 128), (1_000_000, 256))
QUERIES = (128, 2048)
CASES = ("policy_none", "policy_frame", "policy_sets", "retrieval_none", "retrieval_sets")


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, power, clock = (x.strip() for x in q.stdout.splitlines()[0].split(","))
    return {"gpu": name, "power_limit": power, "max_sm_clock": clock}


def timed(fn, warmup, repeats):
    """(times, peak bytes above the inputs during the first call)"""
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.max_memory_allocated()
    fn()
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    for _ in range(warmup):
        fn()
    times = []
    for _ in range(repeats):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        e1.synchronize()
        times.append(e0.elapsed_time(e1) / 1e3)
    return {"time_s_median": statistics.median(times), "time_s_min": min(times), "time_s_max": max(times),
            "repeats": len(times), "peak_bytes_during_call": peak}


def histories(n, items, seed):
    """n long-tailed histories of uniformly drawn ids: (ItemSets on the GPU, lengths)"""
    from recnn_b200.data import ItemSets
    rng = np.random.default_rng(seed)
    lengths = np.minimum(rng.pareto(1.6, n) * 75 + 20, 20000).astype(np.int64)
    lengths[::256] = 8192 + np.arange(len(lengths[::256]))
    offsets = np.concatenate([[0], np.cumsum(lengths)])
    ids = rng.integers(0, items, int(offsets[-1]))
    return ItemSets(torch.from_numpy(ids), torch.from_numpy(offsets), device="cuda"), lengths


def policy_cases(cases, warmup, repeats):
    torch.manual_seed(1)
    with torch.device("cuda"):
        m = recnn_b200.nn.DiscreteActor(S, ITEMS, H)
    param_arena(m)
    out = []
    for N in ROWS:
        state = torch.randn(N, S, device="cuda", generator=torch.Generator(device="cuda").manual_seed(N))
        frame = torch.randint(0, ITEMS, (N, FRAME), device="cuda", generator=torch.Generator(device="cuda").manual_seed(7))
        sets, lengths = histories(N, ITEMS, N) if "policy_sets" in cases else (None, None)
        for k in KS:
            res = {"rows": N, "k": k, "num_items": ITEMS}
            if "policy_none" in cases:
                res["none"] = timed(lambda: m.topk(state, k), warmup, repeats)
            if "policy_frame" in cases:
                res["frame_dense"] = timed(lambda: m.topk(state, k, exclude=frame), warmup, repeats)
            if "policy_sets" in cases:
                res["history_sets"] = timed(lambda: m.topk(state, k, exclude=sets), warmup, repeats)
                res["history_sets"].update(mean_set=float(lengths.mean()), max_set=int(lengths.max()))
            for c in ("frame_dense", "history_sets"):
                if c in res and "none" in res:
                    res[c]["time_ratio_to_none"] = res[c]["time_s_median"] / res["none"]["time_s_median"]
            out.append(res)
            gc.collect()
            torch.cuda.empty_cache()
        del state, frame, sets
    del m
    gc.collect()
    torch.cuda.empty_cache()
    return out


def retrieval_cases(cases, warmup, repeats):
    from recnn_b200.data import ItemIndex
    out = []
    for items, dim in TABLES:
        g = torch.Generator(device="cuda").manual_seed(items)
        table = torch.randn(items, dim, device="cuda", generator=g)
        index = ItemIndex(table, "L2")
        for n in QUERIES:
            q = torch.randn(n, dim, device="cuda", generator=g)
            res = {"items": items, "dim": dim, "queries": n, "k": 10, "metric": "L2"}
            if "retrieval_none" in cases:
                res["none"] = timed(lambda: index.search(q, 10), warmup, repeats)
            if "retrieval_sets" in cases:
                sets, lengths = histories(n, items, n + 1)
                res["history_sets"] = timed(lambda: index.search(q, 10, exclude=sets), warmup, repeats)
                res["history_sets"].update(mean_set=float(lengths.mean()), max_set=int(lengths.max()))
                if "none" in res:
                    res["history_sets"]["time_ratio_to_none"] = (res["history_sets"]["time_s_median"]
                                                                 / res["none"]["time_s_median"])
            out.append(res)
        del index, table
        gc.collect()
        torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--cases", default=",".join(CASES))
    args = ap.parse_args()
    cases = set(args.cases.split(","))
    if not cases <= set(CASES):
        raise SystemExit("--cases takes a comma-separated subset of %s" % ",".join(CASES))
    if not torch.cuda.is_available():
        raise SystemExit("bench_recommend.py needs a GPU")
    result = {"metric": "recommend", **gpu_info(), "S": S, "H": H}
    if cases & {"policy_none", "policy_frame", "policy_sets"}:
        result["policy_topk"] = policy_cases(cases, args.warmup, args.repeats)
    if cases & {"retrieval_none", "retrieval_sets"}:
        result["retrieval"] = retrieval_cases(cases, args.warmup, args.repeats)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
