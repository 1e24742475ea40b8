"""Serving through the DDPG / TD3 critic (Critic.topk / Critic.rank): the actor's candidates or the whole catalogue,
scored by Q on the tensor cores.

Prints one JSON line.  Shapes: the ML-20M critic (S 1290 / A 128 / H 256, 26,744 items) at 128, 2,048 and 16,384 rows
with M = 64 and 1,024 candidates per row and over every item; a 1,000,000 x 256 table (S 2570 / A 256 / H 256) with
candidates only.  k = 10.  Per case: the median / min / max CUDA-event time of one call over --repeats calls after
--warmup calls and the peak torch.cuda.max_memory_allocated() above the inputs during one call (bench_recommend.py's
`timed`), the FLOPs of the call computed from its shapes and their share of the data-sheet dense TF32 rate
(3xTF32: three TF32 products per multiply-add), and rank's time over topk's.  Baselines on the same inputs: the plain
torch composition (critic(state.repeat_interleave(M, 0), table[cand]) then torch.topk) where its [N * M, S + A]
operands fit, and actor + ItemIndex.search(64) for context.  A torch.profiler pass over one call per mode lists the
GEMM kernels the call ran, to show which back end they took.  The card's name, power limit and maximum SM clock are
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
from recnn_b200.data import ItemIndex  # noqa: E402
from recnn_b200.nn.arena import param_arena  # noqa: E402
from bench_recommend import gpu_info, timed  # noqa: E402

K = 10
TF32_DENSE = 495e12          # H100 SXM data sheet, dense TF32, a card allowed 700 W
SHAPES = (
    {"name": "ml20m", "S": 1290, "A": 128, "H": 256, "items": 26_744, "rows": (128, 2048, 16384), "M": (64, 1024),
     "all_items": True},
    {"name": "1m", "S": 2570, "A": 256, "H": 256, "items": 1_000_000, "rows": (128, 2048), "M": (64, 1024),
     "all_items": False},
)
TORCH_FITS = 24e9            # bytes the torch composition may hold at once


def flops(S, A, H, rows, pairs, items=None):
    """TF32 operations of one call: per pair 2AH (candidates; every item: 2AH per item once) + 2H^2 + 2H, per row
    2SH; x3 for 3xTF32"""
    item_term = 2 * A * H * (pairs if items is None else items)
    return 3 * (pairs * (2 * H * H + 2 * H) + rows * 2 * S * H + item_term)


def torch_bytes(S, A, H, pairs):
    # repeated state, its 16-byte-pitch image, the gathered actions and their image, h1, h2, q
    return pairs * (2 * S + 2 * A + 2 * H + 8) * 4


def torch_topk(critic, state, table, cand, k):
    n, m = cand.shape
    q = critic(state.repeat_interleave(m, 0), table[cand.clamp(min=0)].reshape(n * m, -1)).view(n, m)
    q = q.masked_fill(cand < 0, float("-inf"))
    v, j = torch.topk(q, k, dim=1)
    return v, cand.gather(1, j)


def gemm_kernels(fn):
    """names of the GEMM kernels one call runs (torch.profiler, CUDA activities)"""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    names = {}
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA and "gemm" in e.name:
            key = "tc_gemm_kernel" if "tc_gemm_kernel" in e.name else ("gemm_simt" if "simt" in e.name else e.name)
            names[key] = names.get(key, 0) + 1
    return names


def cases(shape, warmup, repeats):
    S, A, H, I = shape["S"], shape["A"], shape["H"], shape["items"]
    torch.manual_seed(1)
    with torch.device("cuda"):
        critic = recnn_b200.nn.Critic(S, A, H).eval()
        actor = recnn_b200.nn.Actor(S, A, H).eval()
    param_arena(critic)
    param_arena(actor)
    g = torch.Generator(device="cuda").manual_seed(I)
    table = torch.randn(I, A, device="cuda", generator=g)
    index = ItemIndex(table, "L2")
    out, profiled = [], {}
    for N in shape["rows"]:
        state = torch.randn(N, S, device="cuda", generator=g)
        res = {"rows": N, "k": K}
        res["actor_search64"] = timed(lambda: index.search(actor(state), 64), warmup, repeats)
        cand64 = index.search(actor(state), 64).id()
        modes = [("cand%d" % m, m) for m in shape["M"]] + ([("all", None)] if shape["all_items"] else [])
        for name, m in modes:
            if m is None:
                cand = None
            elif m == 64:
                cand = cand64
            else:
                base = torch.randint(0, I, (N, 1), device="cuda", generator=g)
                cand = (base + torch.arange(m, device="cuda") * 977) % I     # distinct within a row: 977 is prime to I
            target = (cand64 if cand is None else cand)[:, 7].contiguous()
            pairs = N * (I if m is None else m)
            r = {"pairs": pairs}
            r["topk"] = timed(lambda: critic.topk(state, K, table, candidates=cand), warmup, repeats)
            r["rank"] = timed(lambda: critic.rank(state, target, table, candidates=cand), warmup, repeats)
            r["rank_over_topk"] = r["rank"]["time_s_median"] / r["topk"]["time_s_median"]
            f = flops(S, A, H, N, pairs, I if m is None else None)
            r["tf32_ops"] = f
            r["share_of_dense_tf32"] = f / r["topk"]["time_s_median"] / TF32_DENSE
            if m is not None:
                need = torch_bytes(S, A, H, pairs)
                if need <= TORCH_FITS:
                    r["torch_composition"] = timed(lambda: torch_topk(critic, state, table, cand, K), warmup, repeats)
                    v0, i0 = critic.topk(state, K, table, candidates=cand)
                    v1, i1 = torch_topk(critic, state, table, cand, K)
                    r["torch_max_abs_diff_q"] = float((v0 - v1).abs().max())
                    r["torch_same_ids_rows"] = float((i0 == i1).all(1).float().mean())
                else:
                    r["torch_composition"] = "does not fit: needs %.1f GB" % (need / 1e9)
            else:
                r["torch_composition"] = "does not fit: needs %.1f GB" % (torch_bytes(S, A, H, pairs) / 1e9)
            if name not in profiled and N == shape["rows"][0]:
                profiled[name] = gemm_kernels(lambda: critic.topk(state, K, table, candidates=cand))
            res[name] = r
            del cand
            gc.collect()
            torch.cuda.empty_cache()
        out.append(res)
        del state, cand64
        gc.collect()
        torch.cuda.empty_cache()
    del critic, actor, table, index
    gc.collect()
    torch.cuda.empty_cache()
    return out, profiled


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--repeats", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_critic_serve.py needs a GPU")
    result = {"metric": "critic_serve", **gpu_info(), "k": K, "tf32_dense_datasheet": TF32_DENSE}
    for shape in SHAPES:
        res, prof = cases(shape, args.warmup, args.repeats)
        result[shape["name"]] = {"S": shape["S"], "A": shape["A"], "H": shape["H"], "items": shape["items"],
                                 "cases": res, "gemm_kernels_per_call": prof}
    print(json.dumps(result))


if __name__ == "__main__":
    main()
