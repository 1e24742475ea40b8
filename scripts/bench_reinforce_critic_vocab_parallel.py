"""Vocabulary-parallel item-id REINFORCE critic step at BASELINE configs[4] (S 2570 / H 256 / 1M items), measured on ONE
GPU at 2,048 and 16,384 rows.

Prints one JSON line with, from the same run and for each row count:
  * "single_gpu": the unsharded recnn_discrete_value_step over all 1M items (auto chunk width, built-in SGD);
  * "rank_share": ONE rank's compute at W ranks (default 8, 125,000 local items): recnn_discrete_value_shard_begin,
    merge and end, with the all-gather replaced by local copies of this rank's record (headers fixed up) and the
    all-reduce of the terms left out.  This is a per-rank compute time, NOT an 8-GPU measurement: the exchanges and the
    wait for the slowest rank are not in it;
  * "allreduce_world1": recnn_comm_allreduce of the [2, N, H] terms through a world-1 communicator -- the kernel's
    launch and local copy, not the NVLink transfer of W > 1 ranks;
  * the peak memory above the inputs during each call, and the card's name, power limit and max SM clock.
CUDA-event times: median / min / max over --repeats calls after --warmup calls.
"""
from __future__ import annotations

import argparse
import ctypes
import gc
import json
import os
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
from scripts.bench_reinforce_vocab_parallel import gpu_info, timed, peak_of  # noqa: E402

S, H, I = 2570, 256, 1_000_000


class Step:
    """The nets of `items` items (a rank's block or all of them), a batch of n rows and the step's arguments."""

    def __init__(self, items, n, seed=1):
        torch.manual_seed(seed)
        with torch.device("cuda"):
            self.policy = recnn_b200.nn.DiscreteActor(S, items, H)
            self.value = recnn_b200.nn.Critic(S, items, H, 3e-3)
            self.target = recnn_b200.nn.Critic(S, items, H, 3e-3)
        g = torch.Generator(device="cuda").manual_seed(seed)
        self.batch = {"state": torch.randn(n, S, device="cuda", generator=g),
                      "next_state": torch.randn(n, S, device="cuda", generator=g),
                      "action": torch.randint(0, I, (n,), device="cuda", generator=g),
                      "reward": torch.randn(n, device="cuda", generator=g), "done": torch.zeros(n, device="cuda")}
        self.opt = recnn_b200.optim.SGD(self.value.parameters(), lr=0.0).bind(self.value)
        L = _lib.lib()
        a = self.args = _lib.DiscreteValueArgs()
        a.dims, a.policy_dims = _lib.Dims(S, items, H, 0), self.policy.dims
        a.learn, a.chunk_items, a.n_rows = 1, RF._chunk_items(n, items), n
        b = self.batch
        a.state, a.next_state, a.action = b["state"].data_ptr(), b["next_state"].data_ptr(), b["action"].data_ptr()
        a.reward, a.done = b["reward"].data_ptr(), b["done"].data_ptr()
        a.value = self.opt.c_net(self.value)
        a.target_value = _lib.Net(param_arena(self.target).data_ptr(), None, None, None, None, None)
        a.target_policy = param_arena(self.policy).data_ptr()
        a.value_optim = self.opt.c_optim()
        a.gamma, a.min_value, a.max_value = 0.99, -10.0, 10.0
        self.rng_step = torch.zeros(1, dtype=torch.int64, device="cuda")
        self.losses = torch.zeros(8, device="cuda")
        a.rng_step, a.losses = self.rng_step.data_ptr(), self.losses.data_ptr()
        self.ws_bytes = L.recnn_discrete_value_workspace_bytes(a.dims, a.policy_dims, n, a.chunk_items)
        self.held = {}

    def workspace(self):
        if "ws" not in self.held:
            self.held["ws"] = torch.empty(self.ws_bytes, dtype=torch.uint8, device="cuda")
            self.args.workspace, self.args.workspace_bytes = self.held["ws"].data_ptr(), self.ws_bytes


def single_gpu(n, warmup, repeats):
    L = _lib.lib()
    s = Step(I, n)

    def call():
        s.workspace()
        _lib.check(L.recnn_discrete_value_step(s.args, _lib.stream_ptr()))
    peak = peak_of(call)
    return dict(timed(call, warmup, repeats), chunk_items=s.args.chunk_items, workspace_bytes=s.ws_bytes,
                peak_bytes_during_call=peak, loss=float(s.losses[0]))


def rank_share(n, world, warmup, repeats):
    L = _lib.lib()
    rank = world - 1
    lo, hi = D.vocab_shard(I, rank, world)
    s = Step(hi - lo, n)
    vs = _lib.VocabShard(lo, I, rank, world)
    n_rec = L.recnn_vocab_record_floats(n)

    def call():
        s.workspace()
        if "rec" not in s.held:
            s.held["rec"] = torch.empty(n_rec, device="cuda")
            s.held["gathered"] = torch.empty(world * n_rec, device="cuda")
            s.held["terms"] = torch.empty(2 * n * H, device="cuda")
        rec, gathered, terms = s.held["rec"], s.held["gathered"], s.held["terms"]
        _lib.check(L.recnn_discrete_value_shard_begin(s.args, vs, rec.data_ptr(), _lib.stream_ptr()))
        g = gathered.view(world, n_rec)
        g.copy_(rec.expand(world, n_rec))                 # stands in for the all-gather
        hdr = g[:, :2].view(torch.int32)
        for q in range(world):
            hdr[q] = torch.tensor(D.vocab_shard(I, q, world), dtype=torch.int32)
        _lib.check(L.recnn_discrete_value_shard_merge(s.args, vs, gathered.data_ptr(), terms.data_ptr(),
                                                      _lib.stream_ptr()))
        _lib.check(L.recnn_discrete_value_shard_end(s.args, vs, terms.data_ptr(), _lib.stream_ptr()))
    peak = peak_of(call)
    return dict(timed(call, warmup, repeats), world=world, rank=rank, local_items=hi - lo,
                chunk_items=s.args.chunk_items, workspace_bytes=s.ws_bytes, peak_bytes_during_call=peak,
                error_bits=int(s.losses.view(torch.int32)[4]),
                note="one rank's compute with the exchanges replaced by local copies; not an 8-GPU measurement")


def allreduce_world1(n, warmup, repeats):
    L = _lib.lib()
    floats = 2 * n * H
    h = ctypes.c_void_p()
    _lib.check(L.recnn_comm_create(0, 1, floats, ctypes.byref(h)))
    try:
        mine = ctypes.create_string_buffer(L.recnn_comm_handle_bytes())
        _lib.check(L.recnn_comm_local_handle(h, mine))
        _lib.check(L.recnn_comm_connect(h, mine))
        x = torch.randn(floats, device="cuda")

        def call():
            _lib.check(L.recnn_comm_allreduce(h, x.data_ptr(), floats, _lib.stream_ptr()))
        return dict(timed(call, warmup, repeats), floats=floats, megabytes=floats * 4 / 1e6,
                    note="world 1: launch and local copy, not an NVLink transfer")
    finally:
        torch.cuda.synchronize()
        L.recnn_comm_destroy(h)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--world", type=int, default=8)
    ap.add_argument("--rows", type=int, nargs="+", default=[2048, 16384])
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--repeats", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_reinforce_critic_vocab_parallel.py needs a GPU")
    result = {"metric": "reinforce_critic_vocab_parallel_config4", **gpu_info(), "S": S, "H": H, "num_items": I}
    for n in args.rows:
        res = {}
        for name, fn in (("rank_share", lambda: rank_share(n, args.world, args.warmup, args.repeats)),
                         ("single_gpu", lambda: single_gpu(n, args.warmup, args.repeats)),
                         ("allreduce_world1", lambda: allreduce_world1(n, args.warmup, max(args.repeats, 20)))):
            res[name] = fn()
            gc.collect()
            torch.cuda.empty_cache()
        result["rows_%d" % n] = res
    print(json.dumps(result))


if __name__ == "__main__":
    main()
