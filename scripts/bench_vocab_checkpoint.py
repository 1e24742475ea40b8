"""Full checkpoint of a vocabulary-parallel REINFORCE agent with β, at S 2570 / 2^20 items / H 256, measured at
world 1 on ONE GPU.

The agent (policy, critic and their targets, the built-in Ranger of both) and β (built-in RAdam) are sharded by
enable_vocab_parallel over a one-rank group, their optimizer arenas allocated as after a step.  Timed, host clock
around calls that end in a device synchronisation:
  * "gather": gather_vocab_parallel_state into host memory (the host tensors' allocation included);
  * "load": load_vocab_parallel_state of that checkpoint back into the same agent.
Printed as one JSON line with the bytes each call moves between device and host, the device peak above the resident
arenas during each call, the process's host peak (ru_maxrss) and the card's name and power limit, read in the same
run.  At world 1 every item block is the gathering rank's own: the point-to-point transfer of W > 1 ranks is not
measured here.
"""
from __future__ import annotations

import argparse
import gc
import json
import os
import resource
import subprocess
import sys
import tempfile
import time

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import recnn_b200  # noqa: E402
from recnn_b200 import dist as D  # noqa: E402


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, power = (x.strip() for x in q.stdout.splitlines()[0].split(","))
    return {"gpu": name, "power_limit": power}


def host_peak_gb():
    return resource.getrusage(resource.RUSAGE_SELF).ru_maxrss * 1024 / 1e9


def timed(fn):
    gc.collect()
    torch.cuda.synchronize()
    resident = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    return out, {"wall_s": wall, "device_peak_above_resident_mb": (torch.cuda.max_memory_allocated() - resident) / 2 ** 20,
                 "host_peak_gb": host_peak_gb()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--state-dim", type=int, default=2570)
    ap.add_argument("--items", type=int, default=1 << 20)
    ap.add_argument("--hidden", type=int, default=256)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "the benchmark needs a GPU"
    S, I, H = args.state_dim, args.items, args.hidden
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    with tempfile.TemporaryDirectory() as tmp:
        dist.init_process_group("nccl", init_method="file://" + os.path.join(tmp, "pg"), rank=0, world_size=1,
                                device_id=dev)
        try:
            torch.manual_seed(0)
            with torch.device(dev):
                agent = recnn_b200.nn.Reinforce(recnn_b200.nn.DiscreteActor(S, I, H), recnn_b200.nn.Critic(S, I, H))
                beta = recnn_b200.nn.Beta(S, I)
            agent.to(dev)
            D.enable_vocab_parallel(agent, beta=beta)
            owners = {"policy_optimizer": "policy_net", "value_optimizer": "value_net"}
            for k, opt in agent.optimizers.items():
                opt.c_net(agent.nets[owners[k]])
                opt._t.fill_(1)
            beta.optim.c_net(beta)
            beta.optim._t.fill_(1)
            resident_gb = torch.cuda.memory_allocated() / 1e9
            ckpt, gather = timed(lambda: D.gather_vocab_parallel_state(agent, beta=beta))
            # net state_dicts are views into the full parameter arenas: count each arena once
            moved = sum({t.untyped_storage().data_ptr(): t.untyped_storage().nbytes() for t in _tensors(ckpt)}.values())
            _, load = timed(lambda: D.load_vocab_parallel_state(agent, ckpt, beta=beta))
            gather["bytes"] = load["bytes"] = moved
            vp = agent.nets["policy_net"].__dict__["_recnn_vp"]
            vp.comm.close()
        finally:
            dist.destroy_process_group()
    print(json.dumps(dict(gpu_info(), state_dim=S, items=I, hidden=H, world=1, resident_device_gb=resident_gb,
                          checkpoint_gb=moved / 1e9, gather=gather, load=load,
                          multi_gpu_transfer="not measured: one GPU")))


def _tensors(x):
    if torch.is_tensor(x):
        yield x
    elif isinstance(x, dict):
        for v in x.values():
            yield from _tensors(v)


if __name__ == "__main__":
    main()
