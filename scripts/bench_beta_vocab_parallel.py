"""Vocabulary-parallel behaviour policy beta (recnn_beta_shard_*) at 2^20 items and 2,048 rows, measured on ONE GPU.

Prints one JSON line with, from the same run, at S 1290 and S 2570:
  * "rank_share": ONE rank's compute at W ranks (default 8): recnn_beta_shard_begin + rows + end over its 131,072
    items, with both all-gathers replaced by local copies of the records (the other ranks' records are copies of this
    one's, headers fixed up).  This is a per-rank compute time, NOT an 8-GPU measurement: the exchanges over NVLink
    and the wait for the slowest rank are not in it;
  * "single_gpu": the unsharded recnn_beta_step over all 2^20 items;
  * "allgather_world1": recnn_comm_allgather of one record (4 + 3 x 2,048 floats) through a world-1 communicator --
    the kernel's launch and local copy cost, not the NVLink transfer of W > 1 ranks;
and the card's name, power limit and max SM clock.  Every call uses the built-in RAdam.  Times are CUDA events:
median / min / max over --repeats calls after --warmup calls.  Memory: the peak above what was resident before the
call (the four arenas, the state and the ids), and the whole resident peak.
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
from recnn_b200.nn.update import reinforce as RF  # noqa: E402

I, N = 1 << 20, 2048


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


def memory_of(fn):
    """(peak bytes above what was resident before the call, resident peak) of one call."""
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    fn()
    torch.cuda.synchronize()
    return torch.cuda.max_memory_allocated() - base, torch.cuda.max_memory_allocated()


class Call:
    """recnn_beta_args of one call on a Beta with its built-in RAdam; the workspace is allocated on first use."""

    def __init__(self, beta, state, ids):
        d = beta.dims
        self.chunk = RF._chunk_items(N, d.num_items)
        self.nbytes = _lib.lib().recnn_beta_workspace_bytes(d, N, self.chunk)
        self.beta, self.state, self.ids = beta, state, ids
        self.args = None

    def get(self):
        if self.args is None:
            d = self.beta.dims
            self.probs = torch.empty(N, d.num_items, device="cuda")
            self.loss = torch.empty((), device="cuda")
            self.error = torch.zeros(1, dtype=torch.int32, device="cuda")
            self.ws = torch.empty(self.nbytes, dtype=torch.uint8, device="cuda")
            a = _lib.BetaArgs()
            a.dims, a.n_rows, a.chunk_items = d, N, self.chunk
            a.net, a.optim = self.beta.optim.c_net(self.beta), self.beta.optim.c_optim()
            a.state, a.state_ld = self.state.data_ptr(), self.state.stride(0)
            a.action, a.probs_out = self.ids.data_ptr(), self.probs.data_ptr()
            a.loss, a.error = self.loss.data_ptr(), self.error.data_ptr()
            a.workspace, a.workspace_bytes = self.ws.data_ptr(), self.ws.numel()
            self.args = a
        return self.args


def inputs(S, items, seed=1):
    torch.manual_seed(seed)
    with torch.device("cuda"):
        beta = recnn_b200.nn.Beta(S, items)
    beta.optim.c_net(beta)                              # the moment arenas exist before any measurement
    g = torch.Generator(device="cuda").manual_seed(seed)
    state = torch.randn(N, S, device="cuda", generator=g)
    ids = torch.randint(0, I, (N,), device="cuda", generator=g)
    return beta, state, ids


def single_gpu(S, warmup, repeats):
    beta, state, ids = inputs(S, I)
    c = Call(beta, state, ids)

    def call():
        _lib.check(_lib.lib().recnn_beta_step(c.get(), _lib.stream_ptr()))
    peak, total = memory_of(call)
    res = dict(timed(call, warmup, repeats), chunk_items=c.chunk, peak_bytes_above_resident=peak,
               resident_peak_bytes=total, error=int(c.error), loss=float(c.loss))
    return res


def rank_share(S, world, warmup, repeats):
    L = _lib.lib()
    rank = world - 1
    lo, hi = D.vocab_shard(I, rank, world)
    beta, state, ids = inputs(S, hi - lo)
    c = Call(beta, state, ids)
    vs = _lib.VocabShard(lo, I, rank, world)
    nrec = L.recnn_vocab_record_floats(N)
    held = {}

    def gather(x, out):
        g = out.view(world, nrec)
        g.copy_(x.expand(world, nrec))                   # stands in for the all-gather
        g[:, :2].view(torch.int32).copy_(held["plan"])
        return out

    def call():
        a = c.get()
        if "rec" not in held:
            held["rec"], held["sums"] = torch.empty(nrec, device="cuda"), torch.empty(nrec, device="cuda")
            held["g1"], held["g2"] = torch.empty(world * nrec, device="cuda"), torch.empty(world * nrec, device="cuda")
            held["plan"] = torch.tensor([D.vocab_shard(I, q, world) for q in range(world)], dtype=torch.int32,
                                        device="cuda")
        st = _lib.stream_ptr()
        _lib.check(L.recnn_beta_shard_begin(a, vs, held["rec"].data_ptr(), st))
        g1 = gather(held["rec"], held["g1"])
        _lib.check(L.recnn_beta_shard_rows(a, vs, g1.data_ptr(), held["sums"].data_ptr(), st))
        g2 = gather(held["sums"], held["g2"])
        _lib.check(L.recnn_beta_shard_end(a, vs, g2.data_ptr(), st))
    peak, total = memory_of(call)
    res = dict(timed(call, warmup, repeats), world=world, rank=rank, local_items=hi - lo, chunk_items=c.chunk,
               peak_bytes_above_resident=peak, resident_peak_bytes=total, workspace_bytes=c.nbytes,
               error=int(c.error), loss=float(c.loss),
               note="one rank's compute with the two all-gathers replaced by local copies; not an 8-GPU measurement")
    return res


def allgather_world1(warmup, repeats):
    L = _lib.lib()
    n = L.recnn_vocab_record_floats(N)
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
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--repeats", type=int, default=10)
    ap.add_argument("--state-dims", default="1290,2570")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_beta_vocab_parallel.py needs a GPU")
    result = {"metric": "beta_vocab_parallel", **gpu_info(), "num_items": I, "rows": N}
    for S in (int(x) for x in args.state_dims.split(",")):
        r = {"rank_share": rank_share(S, args.world, args.warmup, args.repeats)}
        gc.collect()
        torch.cuda.empty_cache()
        r["single_gpu"] = single_gpu(S, args.warmup, args.repeats)
        gc.collect()
        torch.cuda.empty_cache()
        result["S%d" % S] = r
    result["allgather_world1"] = allgather_world1(args.warmup, max(args.repeats, 20))
    print(json.dumps(result))


if __name__ == "__main__":
    main()
