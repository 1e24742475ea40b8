"""IVF_PQ search (ItemIndex.build_ivf(nlist, m=M) + search(..., search_param={"nprobe": p, "refine": r})) against
IVF_FLAT over the same lists and the exact flat search, in one session.

Prints one JSON line.  Tables are bench_ivf.py's (imported, not copied): the seeded Gaussian mixture and iid N(0, 1)
rows at 1,000,000 x 256, and the mixture at the ML-20M shape 26,744 x 128.  nlist 1,024, L2, 2,048 queries, k 10.
Per table: the IVF_FLAT build and, per m in {16, 32, 64}, the IVF_PQ build (time from CUDA events around one call) and
index bytes; search times (median / min / max CUDA-event time over --repeats calls after --warmup) and recall@10 against
the flat ids at nprobe 1 / 4 / 16 / 64, for IVF_FLAT and for IVF_PQ at refine 0 and 4.

ADC cost model per call: each work unit (a list and up to TQ of the queries probing it, TQ = 8 / 4 / 2 at m <= 16 / 32
/ 64) reads the list's codes once (code bytes) and the codebooks once (256 x dim x 4 bytes, from L2), and builds TQ
tables of m x 256 entries at 3 x dim / m FLOPs each (table-build FLOPs); every (query, item) pair costs m shared-memory
lookups.  Lookup time is bounded by one shared-memory wavefront per SM per clock: a warp's 32 lookups take as many
wavefronts as the most-used bank has distinct addresses.  With the tables laid out [query][j][256], a lookup's bank is
its code mod 32, so the conflict degree (mean wavefronts per warp lookup) is modelled from the index's own codes for the
scan's mapping (a warp = 32 consecutive items of a list, one subspace j at a time).  It is a model figure, not a
hardware counter: it leaves out the 16-byte code-row loads (2-way conflicted at a 32-byte pitch) and the merge's
shared-memory traffic.  The card's name, power limit and
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
from bench_ivf import HBM, FP32, index_bytes, make_queries, make_table  # noqa: E402
from bench_recommend import gpu_info, timed  # noqa: E402

CASES = (("mixture", 1_000_000, 256), ("iid", 1_000_000, 256), ("mixture", 26_744, 128))
MS, NPROBES, REFINES = (16, 32, 64), (1, 4, 16, 64), (0, 4)
NLIST, NQ, K = 1024, 2048, 10
SMS = 132


def pq_tile(m):
    return 8 if m <= 16 else (4 if m <= 32 else 2)


def built(fn):
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    torch.cuda.synchronize()
    ev[0].record()
    idx = fn()
    ev[1].record()
    ev[1].synchronize()
    return idx, ev[0].elapsed_time(ev[1]) / 1e3


def adc_cost(index, q, nprobe, m):
    iv = index._ivf
    probes = ItemIndex(iv["centroids"], index.metric_name).search(q, nprobe).ids.reshape(-1)
    cnt = torch.bincount(probes, minlength=iv["nlist"]).double()
    lens = (iv["list_offsets"][1:] - iv["list_offsets"][:-1]).double()
    units = torch.ceil(cnt / pq_tile(m))
    pitch = iv["codes"].shape[1]
    return {"code_bytes": float((units * lens).sum()) * pitch,
            "codebook_bytes": float(units.sum()) * 256 * index.dim * 4,
            "table_flops": float(probes.numel()) * 256 * index.dim * 3,
            "lookups": float((cnt * lens).sum()) * m}


def conflict_degree(index, m, groups=8192):
    """mean wavefronts per warp lookup for warps of 32 consecutive items in list order (a sample of groups)"""
    codes = index._ivf["codes"][:, :m].long()
    n = codes.shape[0] // 32 * 32
    g = codes[:n].reshape(-1, 32, m)
    g = g[torch.linspace(0, g.shape[0] - 1, min(groups, g.shape[0]), device=g.device).long()]
    present = torch.zeros(g.shape[0], m, 32, 8, dtype=torch.bool, device=g.device)
    gi = torch.arange(g.shape[0], device=g.device)[:, None, None].expand_as(g)
    ji = torch.arange(m, device=g.device)[None, None, :].expand_as(g)
    present[gi, ji, g % 32, g // 32] = True
    return float(present.sum(-1).amax(-1).float().mean())


def run_case(kind, items, dim, warmup, repeats, clock_hz):
    table, g = make_table(kind, items, dim, items + dim)
    q = make_queries(kind, table, NQ, g)
    flat = ItemIndex(table, "L2")
    exact = flat.search(q, K).ids
    out = {"table": kind, "items": items, "dim": dim, "nlist": NLIST, "queries": NQ, "k": K,
           "flat": timed(lambda: flat.search(q, K), warmup, repeats), "ivf_flat": {}, "ivf_pq": []}
    ivf, t = built(lambda: ItemIndex(table, "L2").build_ivf(NLIST))
    out["ivf_flat"] = {"build_s": t, "index_bytes": index_bytes(ivf), "search": []}
    for p in NPROBES:
        out["ivf_flat"]["search"].append({
            "nprobe": p, "time": timed(lambda: ivf.search(q, K, search_param={"nprobe": p}), warmup, repeats),
            "recall": recall_at_k(ivf.search(q, K, search_param={"nprobe": p}).ids, exact)[1]})
    del ivf
    torch.cuda.empty_cache()
    for m in MS:
        pq, t = built(lambda: ItemIndex(table, "L2").build_ivf(NLIST, m=m))
        r = {"m": m, "build_s": t, "index_bytes": index_bytes(pq),
             "lookup_conflict_degree_model": conflict_degree(pq, m), "search": []}
        for p in NPROBES:
            cost = adc_cost(pq, q, p, m)
            hbm_s = (cost["code_bytes"]) / HBM
            flop_s = cost["table_flops"] / FP32
            lookup_s = cost["lookups"] / 32 * r["lookup_conflict_degree_model"] / (SMS * clock_hz)
            for ref in REFINES:
                sp = {"nprobe": p, "refine": ref}
                s = {"nprobe": p, "refine": ref, "time": timed(lambda: pq.search(q, K, search_param=sp), warmup, repeats),
                     "recall": recall_at_k(pq.search(q, K, search_param=sp).ids, exact)[1]}
                if ref == 0:
                    s.update(cost, hbm_bound_s=hbm_s, fp32_bound_s=flop_s, lookup_bound_s=lookup_s,
                             bound=max((hbm_s, "hbm"), (flop_s, "fp32"), (lookup_s, "smem_lookups"))[1])
                r["search"].append(s)
        out["ivf_pq"].append(r)
        del pq
        torch.cuda.empty_cache()
    del table, flat
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--cases", default="0,1,2", help="indices into CASES")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_ivf_pq.py needs a GPU")
    info = gpu_info()
    clock_hz = float(info["max_sm_clock"].split()[0]) * 1e6
    result = {"metric": "ivf_pq", **info, "cases": [],
              "note": "lookup_conflict_degree_model and lookup_bound_s are modelled from the codes (bank = code mod 32), "
                      "not read from hardware counters"}
    for ci in (int(x) for x in args.cases.split(",")):
        result["cases"].append(run_case(*CASES[ci], args.warmup, args.repeats, clock_hz))
    print(json.dumps(result))


if __name__ == "__main__":
    main()
