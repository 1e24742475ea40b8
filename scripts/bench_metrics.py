"""Exact search under the scipy.spatial.distance metrics that are not inner products (ItemIndex "cityblock",
"chebyshev", "canberra", "braycurtis", "correlation": the CUDA-core distance kernel of csrc/distance.cuh), against the
flat L2 search on the same shape and a torch baseline.

Prints one JSON line.  Shapes: 2,048 and 16,384 queries over a 1,000,000 x 256 table, and 128 and 2,048 queries over
the ML-20M item count, 26,744 x 128; k 10.  Per metric and shape: the median / min / max CUDA-event time of one search
over --repeats calls after --warmup calls and the peak torch.cuda.max_memory_allocated() above the inputs during one
call (bench_recommend.timed), and the achieved FP32 lane-operations per second: n_queries * n_items * dim pair-dims
times the FP32-pipe instructions per pair-dim of the kernel's inner loop (OPS, counted from its SASS), over the time,
beside the H100 SXM data-sheet FP32 issue rate (67 TFLOP/s = 3.35e13 FFMA lane-operations per second at up to 700 W).
That rate bounds the kernel: its shared-memory and HBM traffic per pair-dim is a small fraction of its arithmetic.

The torch baseline: torch.cdist(p=1 / inf) + torch.topk over query slabs for cityblock / chebyshev, and for the others
a broadcast [slab, n_items, dim] composition where a slab of at least 8 queries fits in 2 GB (the 26,744 x 128 table
only); it runs --baseline-repeats times after one warm-up, and is skipped at 16,384 x 1,000,000 x 256, where one run
takes minutes.  Its result is checked against the kernel's: the largest distance difference over the kernel's ids, and
the share of ids both return.  The card's name, power limit and maximum SM clock are read in the same run.
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

from bench_recommend import gpu_info, timed  # noqa: E402
from recnn_b200.data import ItemIndex  # noqa: E402

SHAPES = ((1_000_000, 256, (2048, 16384)), (26_744, 128, (128, 2048)))
K = 10
METRICS = ("cityblock", "chebyshev", "canberra", "braycurtis", "correlation")
# FP32-pipe instructions per pair-dim in the inner loop (cuobjdump -sass of distance_slab_kernel):
#   cityblock   FADD q-t, FADD acc+|.|                                   2
#   chebyshev   FADD q-t, FMNMX.NAN acc,|.|                              2
#   braycurtis  FADD q-t, FADD q+t, two FADD accumulations               4
#   correlation FFMA on the centred values                               1
#   canberra    FADD q-t, FADD |q|+|t|, FSETP den == 0, the IEEE division's five FFMA (reciprocal refinement, quotient,
#               residual, correction), FADD acc; plus MUFU.RCP and FCHK on other pipes and a branch per term   9
OPS = {"cityblock": 2, "chebyshev": 2, "braycurtis": 4, "correlation": 1, "canberra": 9}
FP32_LANE_OPS_PER_S = 3.35e13      # H100 SXM data sheet: 67 TFLOP/s FP32 = 132 SMs x 128 lanes x 1.98 GHz FFMA
SLAB_BYTES = 2 << 30


def torch_distance(q, t, name):
    """[n_q, n_items] distances by a broadcast composition (scipy's formulas, float32)"""
    if name == "cityblock":
        return torch.cdist(q, t, p=1)
    if name == "chebyshev":
        return torch.cdist(q, t, p=float("inf"))
    if name == "correlation":
        qc, tc = q - q.mean(1, keepdim=True), t - t.mean(1, keepdim=True)
        r = (qc @ tc.T) / (qc.norm(dim=1)[:, None] * tc.norm(dim=1)[None, :])
        return (1 - r).clamp(0, 2)
    a, b = q[:, None, :], t[None, :, :]
    if name == "canberra":
        return torch.nan_to_num((a - b).abs() / (a.abs() + b.abs()), nan=0.0).sum(2)
    return (a - b).abs().sum(2) / (a + b).abs().sum(2)


def torch_slab(n_items, dim, name):
    """query rows per slab of the baseline; 0: it does not fit"""
    if name in ("cityblock", "chebyshev", "correlation"):
        return max(1, min(4096, SLAB_BYTES // (4 * n_items)))
    per_query = 4 * n_items * dim * 3                      # the broadcast difference and its temporaries
    s = SLAB_BYTES // per_query
    return int(min(s, 4096)) if s >= 8 else 0


def torch_search(q, t, name, slab):
    ids, dist = [], []
    for r0 in range(0, q.shape[0], slab):
        d, i = torch.topk(torch_distance(q[r0:r0 + slab], t, name), K, dim=1, largest=False)
        ids.append(i)
        dist.append(d)
    return torch.cat(ids), torch.cat(dist)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--baseline-repeats", type=int, default=3)
    ap.add_argument("--metrics", default=",".join(METRICS))
    ap.add_argument("--no-baseline", action="store_true")
    args = ap.parse_args()
    metrics = args.metrics.split(",")
    if not set(metrics) <= set(METRICS):
        raise SystemExit("--metrics takes a comma-separated subset of %s" % ",".join(METRICS))
    if not torch.cuda.is_available():
        raise SystemExit("bench_metrics.py needs a GPU")
    result = {"metric": "retrieval_metrics", **gpu_info(), "k": K, "fp32_lane_ops_per_s_datasheet": FP32_LANE_OPS_PER_S,
              "ops_per_pair_dim": OPS, "cases": []}
    for items, dim, queries in SHAPES:
        g = torch.Generator(device="cuda").manual_seed(items)
        table = torch.randn(items, dim, device="cuda", generator=g)
        for n in queries:
            q = torch.randn(n, dim, device="cuda", generator=g)
            case = {"items": items, "dim": dim, "queries": n, "pair_dims": n * items * dim}
            l2 = ItemIndex(table, "L2")
            case["flat_L2"] = timed(lambda: l2.search(q, K), args.warmup, args.repeats)
            del l2
            for name in metrics:
                index = ItemIndex(table, name)
                r = timed(lambda: index.search(q, K), args.warmup, args.repeats)
                r["fp32_lane_ops_per_s"] = OPS[name] * case["pair_dims"] / r["time_s_median"]
                r["share_of_datasheet_fp32"] = r["fp32_lane_ops_per_s"] / FP32_LANE_OPS_PER_S
                r["time_ratio_to_flat_L2"] = r["time_s_median"] / case["flat_L2"]["time_s_median"]
                slab = torch_slab(items, dim, name)
                if args.no_baseline or slab == 0 or n * items * dim > 2048 * 1_000_000 * 256:
                    r["torch_baseline"] = "not measured: " + ("--no-baseline" if args.no_baseline else
                                                              "does not fit in 2 GB slabs" if slab == 0 else
                                                              "one run takes minutes at this shape")
                else:
                    res = index.search(q, K)
                    b = timed(lambda: torch_search(q, table, name, slab), 1, args.baseline_repeats)
                    bi, bd = torch_search(q, table, name, slab)
                    d_at = torch.gather(torch_distance(q[:1], table, name), 1, res.ids[:1])
                    b.update(query_slab=slab, speedup_of_kernel=b["time_s_median"] / r["time_s_median"],
                             max_abs_dist_diff_row0=float((d_at - res.distances[:1]).abs().max()),
                             max_abs_topk_dist_diff=float((bd - res.distances).abs().max()),
                             id_agreement=float((bi[:, :, None] == res.ids[:, None, :]).any(2).float().mean()))
                    r["torch_baseline"] = b
                case[name] = r
                del index
                gc.collect()
                torch.cuda.empty_cache()
            result["cases"].append(case)
            print(json.dumps(case), file=sys.stderr, flush=True)
        del table
        gc.collect()
        torch.cuda.empty_cache()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
