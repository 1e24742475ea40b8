"""Serving the REINFORCE policy's top-k items at a million-item vocabulary: DiscreteActor.topk (recnn_discrete_topk)
against DiscreteActor.forward + torch.topk, and one rank's share of the vocabulary-parallel call.

Prints one JSON line.  Per case (S 2570 / H 256 / 1,000,000 items, k 10 and 64, rows 1, 128, 2,048 and 16,384): the
median / min / max CUDA-event time of one DiscreteActor.topk call over --repeats calls after --warmup calls, the peak
torch.cuda.max_memory_allocated() above the inputs during one call (its workspace included), and the chunk width the
call picked (recnn_b200.nn.update.reinforce._chunk_items).  Where the dense probabilities fit (rows <= 2,048), the same
for forward + torch.topk, and how many rows return the same ids in the same order (rows may differ where two items'
probabilities round to the same fp32 value, which torch.topk orders as it likes).

FLOPs are the algorithm's, counted from the shapes: 2 N S H for the hidden layer plus 2 N H I for the logits, times 3
for the 3xTF32 passes on the tensor cores.  The share of peak is against NVIDIA's data-sheet dense TF32 rate for the
H100 SXM (495 TFLOP/s), a data-sheet figure for a 700 W card, not a measured one.

The rank share: one rank of W = 8 (125,000 items) runs recnn_discrete_shard_topk, the all-gather is replaced by a local
copy of its record with the other ranks' headers, then recnn_discrete_shard_topk_finish.  It is one GPU's compute, not
an 8-GPU wall time.
"""
from __future__ import annotations

import argparse
import gc
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import recnn_b200  # noqa: E402
from recnn_b200 import _lib  # noqa: E402
from recnn_b200 import dist as D  # noqa: E402
from recnn_b200.nn.arena import param_arena  # noqa: E402
from recnn_b200.nn.update import reinforce as RF  # noqa: E402

TF32_DATASHEET = 495e12
S, H, ITEMS = 2570, 256, 1_000_000
ROWS = (1, 128, 2048, 16384)
KS = (10, 64)
DENSE_MAX_ROWS = 2048
WORLD = 8


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, power, clock = (x.strip() for x in q.stdout.splitlines()[0].split(","))
    return {"gpu": name, "power_limit": power, "max_sm_clock": clock}


def flops(N, I):
    return 3 * (2 * N * S * H + 2 * N * H * I)


def timed(fn, warmup, repeats):
    """(times, peak bytes above the inputs during the first call, last result)"""
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.max_memory_allocated()
    out = fn()
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    for _ in range(warmup):
        out = fn()
    times = []
    for _ in range(repeats):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        out = fn()
        e1.record()
        e1.synchronize()
        times.append(e0.elapsed_time(e1) / 1e3)
    return times, peak, out


def stats(times):
    return {"time_s_median": statistics.median(times), "time_s_min": min(times), "time_s_max": max(times),
            "repeats": len(times)}


def policy(I, seed):
    torch.manual_seed(seed)
    with torch.device("cuda"):
        m = recnn_b200.nn.DiscreteActor(S, I, H)
    param_arena(m)
    return m


def unsharded_cases(warmup, repeats):
    m = policy(ITEMS, 1)
    out = []
    for N in ROWS:
        state = torch.randn(N, S, device="cuda", generator=torch.Generator(device="cuda").manual_seed(N))
        for k in KS:
            times, peak, (v, i) = timed(lambda: m.topk(state, k), warmup, repeats)
            med = statistics.median(times)
            f = flops(N, ITEMS)
            res = {"rows": N, "k": k, "num_items": ITEMS, "chunk_items": RF._chunk_items(N, ITEMS), **stats(times),
                   "peak_bytes_during_call": peak, "flops": f, "tflops_per_s": f / med / 1e12,
                   "share_of_tf32_datasheet": f / med / TF32_DATASHEET}
            if N <= DENSE_MAX_ROWS:
                def dense():
                    p = m(state)
                    return torch.topk(p, k)
                dt, dpeak, (dv, di) = timed(dense, warmup, repeats)
                res["dense"] = {**stats(dt), "peak_bytes_during_call": dpeak}
                res["dense_time_ratio"] = statistics.median(dt) / med
                res["rows_with_same_ids"] = int((di == i).all(1).sum())
                res["rows_with_same_id_sets"] = int((di.sort(1)[0] == i.sort(1)[0]).all(1).sum())
                del dv, di
            out.append(res)
            del v, i
            gc.collect()
            torch.cuda.empty_cache()
        del state
    del m
    gc.collect()
    torch.cuda.empty_cache()
    return out


def rank_share_cases(warmup, repeats):
    L = _lib.lib()
    rank = WORLD - 1
    lo, hi = D.vocab_shard(ITEMS, rank, WORLD)
    m = policy(hi - lo, 2)
    d = m.dims
    vs = _lib.VocabShard(lo, ITEMS, rank, WORLD)
    st = _lib.stream_ptr()
    heads = torch.tensor([D.vocab_shard(ITEMS, q, WORLD) for q in range(WORLD)], dtype=torch.int32, device="cuda")
    out = []
    for N in (2048, 16384):
        state = torch.randn(N, S, device="cuda", generator=torch.Generator(device="cuda").manual_seed(N))
        for k in KS:
            chunk = RF._chunk_items(N, d.num_items)
            nbytes = L.recnn_discrete_topk_workspace_bytes(d, N, k, chunk)

            def call():
                ws = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
                rec = torch.empty(L.recnn_vocab_topk_record_floats(N, k), device="cuda")
                _lib.check(L.recnn_discrete_shard_topk(d, vs, param_arena(m).data_ptr(), state.data_ptr(), N, k, None,
                                                       0, chunk, rec.data_ptr(), ws.data_ptr(), nbytes, st))
                del ws
                gathered = rec.repeat(WORLD)
                gathered.view(WORLD, -1)[:, :2].view(torch.int32).copy_(heads)
                values = torch.empty(N, k, device="cuda")
                ids = torch.empty(N, k, dtype=torch.int64, device="cuda")
                flag = torch.empty(1, dtype=torch.int32, device="cuda")
                _lib.check(L.recnn_discrete_shard_topk_finish(d, vs, gathered.data_ptr(), N, k, None, 0,
                                                              values.data_ptr(), ids.data_ptr(), flag.data_ptr(), st))
                return flag
            times, peak, flag = timed(call, warmup, repeats)
            med = statistics.median(times)
            f = flops(N, hi - lo)
            out.append({"world": WORLD, "rank": rank, "local_items": hi - lo, "rows": N, "k": k, "chunk_items": chunk,
                        **stats(times), "peak_bytes_during_call": peak, "flops": f, "tflops_per_s": f / med / 1e12,
                        "share_of_tf32_datasheet": f / med / TF32_DATASHEET, "error_bits": int(flag.item())})
        del state
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--repeats", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_policy_topk.py needs a GPU")
    result = {"metric": "policy_topk", **gpu_info(), "tf32_datasheet_flops": TF32_DATASHEET, "S": S, "H": H}
    result["cases"] = unsharded_cases(args.warmup, args.repeats)
    result["rank_share"] = rank_share_cases(args.warmup, args.repeats)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
