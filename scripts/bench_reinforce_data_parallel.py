"""Data-parallel REINFORCE (recnn_b200.dist.enable_data_parallel on a DiscreteActor agent) at the Top-K notebook's
shape: S 1290, H 2048, 5,000 items, K 10, policy_step 10, Top-K correction with a data-parallel Beta; one-hot and
item-id batch actions.

Prints one JSON line with, from the same run and for each action form:
  * "single_gpu": Reinforce.update() calls/s of the unsharded agent at 128 and at 1,024 rows per env step;
  * "rank_share": ONE rank's share at W ranks (default 8): 128 of 1,024 rows per env step, the rank's compute with every
    exchange replaced by a local copy (an all-gather repeats this rank's tensor W times, a row record's header
    re-numbered to rank q's rows; the all-reduces are left out).  A per-rank compute rate, NOT a W-GPU measurement: the
    transfers and the wait for the slowest rank are not in it;
  * "processes": the wall-clock calls/s of W processes, one per GPU, each on its 1,024 / W rows (only when at least 2
    GPUs exist; W = the GPU count, at most --world);
  * "exchange_bytes": the bytes each exchange of one rank moves per call, computed from the shapes;
  * the card's name, power limit and max SM clock, read in the same run.
Host-clock times around calls that end in a device synchronise (every update reads its losses back): median over
--repeats windows of --calls calls after --warmup calls.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import recnn_b200  # noqa: E402
from recnn_b200 import _lib  # noqa: E402
from recnn_b200 import dist as D  # noqa: E402
from recnn_b200.nn.arena import param_arena  # noqa: E402
from scripts.bench_reinforce_vocab_parallel import gpu_info  # noqa: E402

S, H, I, K, POLICY_STEP = 1290, 2048, 5000, 10, 10


def make_agent(dev, seed=1):
    torch.manual_seed(seed)
    agent = recnn_b200.nn.Reinforce(recnn_b200.nn.DiscreteActor(S, I, H),
                                    recnn_b200.nn.Critic(S, I, H, 3e-3)).to(torch.device(dev))
    agent.params.update(K=K, policy_step=POLICY_STEP, reinforce=recnn_b200.nn.ChooseREINFORCE(
        recnn_b200.nn.ChooseREINFORCE.reinforce_with_TopK_correction))
    beta = recnn_b200.nn.Beta(S, I).to(dev)
    pol = agent.nets["policy_net"]

    def select(state, action, K, writer, step, **kwargs):
        return pol._select_action_with_TopK_correction(state, beta.forward, action, K=K, writer=writer, step=step)
    pol.select_action = select
    return agent, beta


def batches(form, n, dev, count=8, seed=2):
    g = torch.Generator(device=dev).manual_seed(seed)
    out = []
    for _ in range(count):
        ids = torch.randint(0, I, (n,), device=dev, generator=g)
        action = ids if form == "ids" else torch.nn.functional.one_hot(ids, I).float()
        out.append({"state": torch.randn(n, S, device=dev, generator=g), "action": action,
                    "reward": torch.randint(-2, 3, (n,), device=dev, generator=g).float(),
                    "next_state": torch.randn(n, S, device=dev, generator=g), "done": torch.zeros(n, device=dev)})
    return out


def rate(agent, bs, warmup, calls, repeats):
    def run(k):
        for _ in range(k):
            agent.update(bs[agent._step % len(bs)])
            agent.step()
    run(warmup)
    rates = []
    for _ in range(repeats):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        run(calls)
        torch.cuda.synchronize()
        rates.append(calls / (time.perf_counter() - t0))
    return {"calls_per_s_median": statistics.median(rates), "calls_per_s_min": min(rates),
            "calls_per_s_max": max(rates), "windows": repeats, "calls_per_window": calls}


class LocalCopies:
    """One rank's communicator with the other ranks replaced by local copies of this rank's tensors (see above)."""
    capacity = 1 << 62

    def __init__(self, world, record_floats):
        self.world, self.record_floats = world, record_floats

    def all_gather(self, t):
        out = t.reshape(-1).repeat(self.world)
        if t.dtype == torch.float32 and t.numel() == self.record_floats:
            hdr = out.view(self.world, -1)[:, :4].view(torch.int32)
            n = int(hdr[0, 1])
            hdr[:, 0] = torch.arange(self.world, device=t.device, dtype=torch.int32) * n
        return out

    def all_reduce(self, t):
        return t

    def close(self):
        pass


def exchange_bytes(form, n_rank, world):
    L = _lib.lib()
    d = _lib.Dims(S, I, H, 0)
    f = 4
    out = {"row_counts_all_gather": world * f,
           "reward_rows_all_gather": world * n_rank * f,
           "beta_grad_all_reduce": (I * ((S + 3) // 4 * 4) + I + 2) * f,
           "policy_grad_all_reduce_per_policy_step": (int(param_arena(recnn_b200.nn.DiscreteActor(S, I, H)).numel())
                                                      + 2) * f}
    if form == "ids":
        out["critic_grad_all_reduce"] = int(L.recnn_discrete_value_dp_grad_floats(d)) * f
        out["critic_rows_all_gather"] = world * int(L.recnn_discrete_value_dp_record_floats(d, n_rank)) * f
    else:
        out["critic_grad_all_reduce"] = (H * ((S + I + 3) // 4 * 4) + H + H * H + H + H + 1 + 1) * f
    return out


def _mp_worker(rank, world, form, n_global, warmup, calls, repeats, q):
    import torch.distributed as dist
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    try:
        dev = "cuda:%d" % rank
        agent, beta = make_agent(dev)
        D.enable_data_parallel(agent, beta=beta)
        lo, hi = D.shard_rows(n_global, rank, world)
        bs = [{k: v[lo:hi].contiguous() for k, v in b.items()} for b in batches(form, n_global, dev)]
        r = rate(agent, bs, warmup, calls, repeats)
        q.put(r if rank == 0 else None)
        D.row_parallel_of(agent.nets["policy_net"]).comm.close()
    finally:
        dist.destroy_process_group()


def processes(form, world, n_global, warmup, calls, repeats):
    import torch.multiprocessing as mp
    import socket
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(s.getsockname()[1])
    s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_mp_worker, args=(r, world, form, n_global, warmup, calls, repeats, q))
             for r in range(world)]
    for p in procs:
        p.start()
    res = [q.get(timeout=1800) for _ in range(world)]
    for p in procs:
        p.join(timeout=600)
    return next(r for r in res if r is not None)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--world", type=int, default=8)
    ap.add_argument("--rows", type=int, default=1024, help="rows per env step of the whole batch")
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--forms", default="ids,onehot")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_reinforce_data_parallel measures on the GPU; no CUDA device found")
    out = {"shape": {"S": S, "H": H, "num_items": I, "K": K, "policy_step": POLICY_STEP, "method": "TopK + Beta"},
           "world": args.world, "rows_per_env_step": args.rows}
    out.update(gpu_info())
    n_rank = -(-args.rows // args.world)
    L = _lib.lib()
    for form in args.forms.split(","):
        res = {"single_gpu": {}}
        for n in (128, args.rows):
            agent, beta = make_agent("cuda")
            res["single_gpu"][str(n)] = rate(agent, batches(form, n, "cuda"), args.warmup, args.calls, args.repeats)
            del agent, beta
            torch.cuda.empty_cache()
        agent, beta = make_agent("cuda")
        comm = LocalCopies(args.world, int(L.recnn_discrete_value_dp_record_floats(_lib.Dims(S, I, H, 0), n_rank)))
        D.data_parallel_in_place(agent.nets, D.RowParallel(None, 0, args.world, comm), beta, agent.optimizers)
        res["rank_share"] = dict(rate(agent, batches(form, n_rank, "cuda"), args.warmup, args.calls, args.repeats),
                                 rows=n_rank, note="one rank's compute, exchanges replaced by local copies; not a "
                                                   "%d-GPU measurement" % args.world)
        del agent, beta
        torch.cuda.empty_cache()
        gpus = min(torch.cuda.device_count(), args.world)
        res["processes"] = (dict(processes(form, gpus, args.rows, args.warmup, args.calls, args.repeats), world=gpus)
                            if gpus >= 2 else "not measured: %d GPU(s)" % torch.cuda.device_count())
        res["exchange_bytes"] = exchange_bytes(form, n_rank, args.world)
        out[form] = res
    print(json.dumps(out))


if __name__ == "__main__":
    main()
