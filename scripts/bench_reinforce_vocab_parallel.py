"""Vocabulary-parallel REINFORCE policy update at BASELINE configs[4] (S 2570 / H 256 / 1M items / 163,840 saved rows =
16,384 x policy_step 10), measured on ONE GPU.

Prints one JSON line with, from the same run:
  * "single_gpu": the unsharded recnn_reinforce_policy_grad_chunked call over all 1M items (auto chunk width);
  * "rank_share": ONE rank's compute at W ranks (default 8): recnn_reinforce_shard_stats + recnn_reinforce_shard_grad
    over its 125,000 items, with the all-gather replaced by a local copy of the records (the other ranks' records are
    copies of this one's, headers fixed up).  This is a per-rank compute time, NOT an 8-GPU measurement: the exchanges
    and the wait for the slowest rank are not in it;
  * "allgather_world1": recnn_comm_allgather of one record (4 + 3 x 163,840 floats) through a world-1 communicator --
    the kernel's launch and local copy cost, not the NVLink transfer of W > 1 ranks;
  * the card's name, power limit and max SM clock, and the per-rank peak memory above the inputs.
CUDA-event times: median / min / max over --repeats calls after --warmup calls.
"""
from __future__ import annotations

import argparse
import ctypes
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

S, H, I, R = 2570, 256, 1_000_000, 163_840


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, power, clock = (x.strip() for x in q.stdout.splitlines()[0].split(","))
    return {"gpu": name, "power_limit": power, "max_sm_clock": clock}


def timed(fn, warmup, repeats):
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
            "repeats": len(times)}


def peak_of(fn):
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.max_memory_allocated()
    fn()
    torch.cuda.synchronize()
    return torch.cuda.max_memory_allocated() - base


def inputs(items, seed=1):
    torch.manual_seed(seed)
    with torch.device("cuda"):
        m = recnn_b200.nn.DiscreteActor(S, items, H)
    g = torch.Generator(device="cuda").manual_seed(seed)
    state = torch.randn(R, S, device="cuda", generator=g)
    action = torch.randint(0, I, (R,), device="cuda", generator=g)
    blp = torch.log(torch.empty(R, device="cuda").uniform_(0.5 / I, 2.0 / I, generator=g))
    ret = torch.randn(R, device="cuda", generator=g)
    return m, state, action, blp, ret


def single_gpu(warmup, repeats):
    L = _lib.lib()
    m, state, action, blp, ret = inputs(I)
    d = m.dims
    chunk = RF._chunk_items(R, I)
    flat = param_arena(m)
    grads = torch.zeros_like(flat)
    out = torch.zeros(2, device="cuda")
    held = {}

    def call():
        if "scratch" not in held:
            held["scratch"] = torch.empty(L.recnn_reinforce_scratch_floats(d, R, chunk), device="cuda")
        _lib.check(L.recnn_reinforce_policy_grad_chunked(d, flat.data_ptr(), grads.data_ptr(), state.data_ptr(),
                                                         action.data_ptr(), blp.data_ptr(), ret.data_ptr(), R,
                                                         _lib.REINFORCE_TOPK, 10, chunk, out.data_ptr(),
                                                         held["scratch"].data_ptr(), _lib.stream_ptr()))
    peak = peak_of(call)
    res = dict(timed(call, warmup, repeats), chunk_items=chunk, n_chunks=-(-I // chunk), peak_bytes_during_call=peak,
               loss=float(out[0]))
    return res


def rank_share(world, warmup, repeats):
    L = _lib.lib()
    rank = world - 1
    lo, hi = D.vocab_shard(I, rank, world)
    m, state, action, blp, ret = inputs(hi - lo)
    d = m.dims
    chunk = RF._chunk_items(R, d.num_items)
    flat = param_arena(m)
    grads = torch.zeros_like(flat)
    out = torch.zeros(3, device="cuda")
    vs = _lib.VocabShard(lo, I, rank, world)
    n_rec = L.recnn_vocab_record_floats(R)
    held = {}

    def call():
        if "scratch" not in held:
            held["scratch"] = torch.empty(L.recnn_reinforce_scratch_floats(d, R, chunk), device="cuda")
            held["rec"] = torch.empty(n_rec, device="cuda")
            held["gathered"] = torch.empty(world * n_rec, device="cuda")
        rec, gathered = held["rec"], held["gathered"]
        _lib.check(L.recnn_reinforce_shard_stats(d, vs, flat.data_ptr(), state.data_ptr(), action.data_ptr(), R, chunk,
                                                 rec.data_ptr(), held["scratch"].data_ptr(), _lib.stream_ptr()))
        g = gathered.view(world, n_rec)
        g.copy_(rec.expand(world, n_rec))                 # stands in for the all-gather
        hdr = g[:, :2].view(torch.int32)
        for q in range(world):
            hdr[q] = torch.tensor(D.vocab_shard(I, q, world), dtype=torch.int32)
        _lib.check(L.recnn_reinforce_shard_grad(d, vs, flat.data_ptr(), grads.data_ptr(), state.data_ptr(),
                                                action.data_ptr(), blp.data_ptr(), ret.data_ptr(), R,
                                                _lib.REINFORCE_TOPK, 10, chunk, gathered.data_ptr(), out.data_ptr(),
                                                held["scratch"].data_ptr(), _lib.stream_ptr()))
    peak = peak_of(call)
    res = dict(timed(call, warmup, repeats), world=world, rank=rank, local_items=hi - lo, chunk_items=chunk,
               n_chunks=-(-(hi - lo) // chunk), peak_bytes_during_call=peak,
               flags=out.view(torch.int32)[1:].tolist(),
               note="one rank's compute with the exchanges replaced by local copies; not an 8-GPU measurement")
    return res


def allgather_world1(warmup, repeats):
    L = _lib.lib()
    n = L.recnn_vocab_record_floats(R)
    h = ctypes.c_void_p()
    _lib.check(L.recnn_comm_create(0, 1, n, ctypes.byref(h)))
    try:
        mine = ctypes.create_string_buffer(L.recnn_comm_handle_bytes())
        _lib.check(L.recnn_comm_local_handle(h, mine))
        _lib.check(L.recnn_comm_connect(h, mine))
        x = torch.randn(n, device="cuda")
        y = torch.empty(n, device="cuda")

        def call():
            _lib.check(L.recnn_comm_allgather(h, x.data_ptr(), n, y.data_ptr(), _lib.stream_ptr()))
        res = dict(timed(call, warmup, repeats), floats=n)
        torch.cuda.synchronize()
        res["bit_exact"] = bool(torch.equal(x.view(torch.int32), y.view(torch.int32)))
        return res
    finally:
        torch.cuda.synchronize()
        L.recnn_comm_destroy(h)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--world", type=int, default=8)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--repeats", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_reinforce_vocab_parallel.py needs a GPU")
    result = {"metric": "reinforce_vocab_parallel_config5", **gpu_info(), "S": S, "H": H, "num_items": I, "rows": R}
    result["rank_share"] = rank_share(args.world, args.warmup, args.repeats)
    gc.collect()
    torch.cuda.empty_cache()
    result["single_gpu"] = single_gpu(args.warmup, args.repeats)
    gc.collect()
    torch.cuda.empty_cache()
    result["allgather_world1"] = allgather_world1(args.warmup, max(args.repeats, 20))
    print(json.dumps(result))


if __name__ == "__main__":
    main()
