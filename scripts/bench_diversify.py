"""Diversified re-ranking (recnn_b200.utils.diversify): greedy MMR and greedy DPP over each row's candidate pool, one
kernel that reads every candidate's row from the resident table once.

Prints one JSON line.  Shapes: N in {128, 2,048, 16,384} pools x m in {64, 256} candidates x k in {10, 64} picks, both
methods at weight 0.5, over a 26,744 x 128 table (the ML-20M catalogue at dim 128) and a 1,000,000 x 256 table; pool
ids drawn uniformly (about 1% padding), scores standard normal.  Per case: the median / min / max CUDA-event time of
one `diversify` call over --repeats calls after --warmup calls (it includes the call's one read-back of the error
flag), the peak torch.cuda.max_memory_allocated() above the inputs during one call, and the cost model: bytes N m D 4
of candidate rows, FP32 FLOPs N (2 m D (k + 1) + DPP m k^2), the least time the H100 SXM data sheet allows for them
(3.35 TB/s, 67 TFLOP/s dense FP32, a card allowed 700 W) and the call's share of it.  Baseline on the same inputs: a
batched torch composition (`table[ids]`, normalised, then k steps of a batched GEMV and the greedy update), its time
and peak, and the share of slate ids on which the two agree (ties and fp32 rounding may order near-equal items
differently).  The card's name, power limit and maximum SM clock are read in the same run.
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

from recnn_b200.utils import diversify  # noqa: E402
from bench_recommend import gpu_info, timed  # noqa: E402

TABLES = ((26_744, 128), (1_000_000, 256))
ROWS, POOLS, KS = (128, 2048, 16384), (64, 256), (10, 64)
WEIGHT = 0.5
HBM = 3.35e12                # H100 SXM data sheet, bytes/s
FP32 = 67e12                 # H100 SXM data sheet, dense FP32 FLOP/s


def cost(n, m, d, k, method):
    return n * m * d * 4, n * (2 * m * d * (k + 1) + (m * k * k if method == "dpp" else 0))


def torch_composition(ids, scores, table, k, method, w):
    n, m = ids.shape
    x = table[ids.clamp(min=0)]
    xn = torch.nn.functional.normalize(x, dim=2)
    alive = ids >= 0
    rows = torch.arange(n, device=ids.device)
    out = torch.full((n, k), -1, dtype=torch.int64, device=ids.device)
    neg = torch.tensor(-float("inf"), device=ids.device)
    if method == "mmr":
        ms = torch.zeros(n, m, device=ids.device)
    else:
        a2 = w / (1 - w)
        d2 = torch.ones(n, m, device=ids.device)
        c = torch.zeros(n, m, k, device=ids.device)
    done = torch.zeros(n, dtype=torch.bool, device=ids.device)
    for t in range(k):
        if method == "mmr":
            obj = w * scores - (1 - w) * ms
        else:
            obj = a2 * scores + torch.log(d2.clamp(min=0))
        obj = torch.where(alive, obj, neg)
        j = obj.argmax(1)
        ok = alive[rows, j] & ~done
        if method == "dpp":
            ok &= d2[rows, j] >= 1e-4
        done |= ~ok
        cid = ids[rows, j]
        out[:, t] = torch.where(ok, cid, -1)
        sim = torch.bmm(xn, xn[rows, j].unsqueeze(2)).squeeze(2).clamp(-1, 1)
        if method == "mmr":
            ms = torch.where(torch.full_like(ms, t == 0, dtype=torch.bool), sim, torch.maximum(ms, sim))
        else:
            e = (0.5 * (1 + sim) - (c[:, :, :t] * c[rows, j, :t].unsqueeze(1)).sum(2)) / d2[rows, j].clamp(min=1e-30).sqrt().unsqueeze(1)
            c[:, :, t] = e
            d2 = d2 - e * e
        alive &= ids != cid.unsqueeze(1)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--repeats", type=int, default=10)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_diversify.py needs a GPU")
    result = {"metric": "diversify", **gpu_info(), "weight": WEIGHT, "hbm_datasheet": HBM,
              "fp32_dense_datasheet": FP32, "cases": []}
    g = torch.Generator(device="cuda").manual_seed(0)
    for items, D in TABLES:
        table = torch.randn(items, D, device="cuda", generator=g)
        for N in ROWS:
            for m in POOLS:
                ids = torch.randint(-items // 100, items, (N, m), device="cuda", generator=g).clamp(min=-1)
                scores = torch.randn(N, m, device="cuda", generator=g)
                for k in KS:
                    for method in ("mmr", "dpp"):
                        byt, fl = cost(N, m, D, k, method)
                        bound = max(byt / HBM, fl / FP32)
                        r = {"items": items, "dim": D, "rows": N, "m": m, "k": k, "method": method, "bytes": byt,
                             "flops": fl, "bound_s": bound, "bound_by": "bytes" if byt / HBM >= fl / FP32 else "flops"}
                        r["call"] = timed(lambda: diversify(ids, scores, table, k, method, WEIGHT), args.warmup,
                                          args.repeats)
                        r["share_of_bound"] = bound / r["call"]["time_s_median"]
                        r["torch_composition"] = timed(lambda: torch_composition(ids, scores, table, k, method, WEIGHT),
                                                       1, 3)
                        got = diversify(ids, scores, table, k, method, WEIGHT)[0]
                        ref = torch_composition(ids, scores, table, k, method, WEIGHT)
                        r["agreement_with_torch"] = float((got == ref).double().mean())
                        result["cases"].append(r)
                        print(json.dumps(r), file=sys.stderr)
                        del got, ref
                        gc.collect()
                        torch.cuda.empty_cache()
                del ids, scores
        del table
        gc.collect()
        torch.cuda.empty_cache()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
