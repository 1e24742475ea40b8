"""Slate diversity (recnn_b200.utils.metrics.slate_distances): pairwise distances within each served slate, read from
the resident table by one kernel.

Prints one JSON line.  Shapes: N in {128, 2,048, 16,384} rows x k in {10, 64} slots x D in {128, 256} over a
1,000,000-item table, ids drawn uniformly (about 1% empty slots), both metrics.  Per case: the median / min / max
CUDA-event time of one `slate_distances` call over --repeats calls after --warmup calls (it includes the call's one
read-back of the error flag) and of the bare kernel launch through the C entry point, the peak
torch.cuda.max_memory_allocated() above the inputs during one call (bench_recommend.py's `timed`), and the cost model:
bytes N k D 4 of gathered rows, FLOPs N k(k-1)/2 3D, the least time the H100 SXM data sheet allows for them (3.35 TB/s,
67 TFLOP/s dense FP32, a card allowed 700 W) and the kernel's share of it.  Baseline on the same inputs: the torch
composition (`torch.cdist` on `table[ids]`, or normalised rows' products for cosine, then the same masked reductions)
and its largest difference from the kernel.  The card's name, power limit and maximum SM clock are read in the same
run.
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

from recnn_b200 import _lib  # noqa: E402
from recnn_b200.utils.metrics import slate_distances  # noqa: E402
from bench_recommend import gpu_info, timed  # noqa: E402

ITEMS = 1_000_000
ROWS, KS, DIMS = (128, 2048, 16384), (10, 64), (128, 256)
HBM = 3.35e12                # H100 SXM data sheet, bytes/s
FP32 = 67e12                 # H100 SXM data sheet, dense FP32 FLOP/s
TORCH_FITS = 24e9            # bytes the torch composition may hold at once


def cost(n, k, d):
    return n * k * d * 4, n * k * (k - 1) // 2 * 3 * d


def torch_composition(ids, table, metric):
    x = table[ids.clamp(min=0)]
    if metric == "euclidean":
        m = torch.cdist(x, x)
    else:
        xn = torch.nn.functional.normalize(x, dim=2)
        m = (1 - xn @ xn.transpose(1, 2)).clamp(0, 2)
    f = ids >= 0
    pair = f[:, :, None] & f[:, None, :] & torch.ones(ids.shape[1], ids.shape[1], dtype=torch.bool,
                                                      device=ids.device).triu(1)
    c = f.sum(1)
    npairs = (c * (c - 1) // 2).double()
    mean = torch.where(pair, m, 0).double().sum((1, 2)) / npairs
    mn = torch.where(pair, m, float("inf")).amin((1, 2))
    return mean.float(), torch.where(c >= 2, mn, float("nan"))


def raw_call(ids, table, metric):
    """the bare kernel: outputs allocated once, no read-back"""
    n, k = ids.shape
    mean, mn = torch.empty(n, device="cuda"), torch.empty(n, device="cuda")
    count, flag = torch.empty(n, dtype=torch.int32, device="cuda"), torch.empty(1, dtype=torch.int32, device="cuda")
    L = _lib.lib()
    m = 0 if metric == "euclidean" else 1
    stream = _lib.stream_ptr()

    def go():
        _lib.check(L.recnn_slate_distances(ids.data_ptr(), n, k, table.data_ptr(), table.shape[0], table.shape[1], m,
                                           mean.data_ptr(), mn.data_ptr(), count.data_ptr(), None, flag.data_ptr(),
                                           stream))
    return go


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--repeats", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_slate.py needs a GPU")
    result = {"metric": "slate_distances", **gpu_info(), "items": ITEMS, "hbm_datasheet": HBM,
              "fp32_dense_datasheet": FP32, "cases": []}
    g = torch.Generator(device="cuda").manual_seed(0)
    for D in DIMS:
        table = torch.randn(ITEMS, D, device="cuda", generator=g)
        for N in ROWS:
            for k in KS:
                ids = torch.randint(-ITEMS // 100, ITEMS, (N, k), device="cuda", generator=g).clamp(min=-1)
                byt, fl = cost(N, k, D)
                bound = max(byt / HBM, fl / FP32)
                for metric in ("euclidean", "cosine"):
                    r = {"rows": N, "k": k, "dim": D, "metric": metric, "bytes": byt, "flops": fl,
                         "bound_s": bound, "bound_by": "bytes" if byt / HBM >= fl / FP32 else "flops"}
                    r["call"] = timed(lambda: slate_distances(ids, table, metric), args.warmup, args.repeats)
                    r["kernel"] = timed(raw_call(ids, table, metric), args.warmup, args.repeats)
                    r["kernel_share_of_bound"] = bound / r["kernel"]["time_s_median"]
                    if byt + N * k * k * 4 * 3 <= TORCH_FITS:
                        r["torch_composition"] = timed(lambda: torch_composition(ids, table, metric), args.warmup,
                                                       args.repeats)
                        m0, n0, _ = slate_distances(ids, table, metric)
                        m1, n1 = torch_composition(ids, table, metric)
                        r["torch_max_abs_diff_mean"] = float((m0 - m1).abs().nan_to_num(0).max())
                        r["torch_max_abs_diff_min"] = float((n0 - n1).abs().nan_to_num(0).max())
                    else:
                        r["torch_composition"] = "does not fit"
                    result["cases"].append(r)
                    gc.collect()
                    torch.cuda.empty_cache()
                del ids
        del table
        gc.collect()
        torch.cuda.empty_cache()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
