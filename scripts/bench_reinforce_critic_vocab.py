"""REINFORCE critic at large vocabularies: value_update with item-id actions (recnn_discrete_value_step), and one full
reinforce_update policy step.

Prints one JSON line.  Per config: the median / min / max CUDA-event time of one call over --repeats calls after
--warmup calls, and the peak torch.cuda.max_memory_allocated() during the first call above the memory in use before it
(the nets, their gradient and optimizer arenas already exist; the call's workspace is allocated in it).

FLOPs are the algorithm's, counted from the shapes, times 3 for the 3xTF32 passes on the tensor cores.  For one
value_update in item-id mode (N rows, state S, critic hidden H, policy hidden Hp, I items):
  2 N (S Hp + Hp I + I H)    target policy layer 1, its logits, the projection of its softmax on the critic's W1a
  2 N (2 S H + 2 H H)        target and online critic layers 1 (state block) and 2
  2 N (S H + 2 H H)          dW1 (state block), dW2 and dz1
The share of peak is against NVIDIA's data-sheet dense TF32 rate for the H100 SXM (495 TFLOP/s), a data-sheet figure for a
700 W card, not a measured one.

Configs (S / H / num_items / N):
  A  1290 / 256 / 5,000     / 1,280    item ids vs the dense one-hot on the same seeded inputs (loss and weight difference)
  B  2570 / 256 / 1,048,576 / 2,048    one GPU's share of BASELINE configs[4]'s batch
  C  2570 / 256 / 1,048,576 / 16,384   the whole configs[4] batch
  D  2570 / 256 / 1,048,576 / 2,048    one reinforce_update policy step (policy_step 10: the gradient runs over 20,480 saved
                                       rows), with select_action's dense probabilities (the reference's API)
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
from recnn_b200.nn.update import reinforce as RF  # noqa: E402

TF32_DATASHEET = 495e12
CONFIGS = {"A": (1290, 256, 5_000, 1_280), "B": (2570, 256, 1 << 20, 2_048), "C": (2570, 256, 1 << 20, 16_384),
           "D": (2570, 256, 1 << 20, 2_048)}


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, power, clock = (x.strip() for x in q.stdout.splitlines()[0].split(","))
    return {"gpu": name, "power_limit": power, "max_sm_clock": clock}


def value_flops(S, H, Hp, I, N):
    return 3 * 2 * N * (S * Hp + Hp * I + I * H + 3 * S * H + 4 * H * H)


def policy_step_flops(S, H, I, N, steps):
    R = N * steps
    chunk = RF._chunk_items(R, I)
    n_chunks = -(-I // chunk)
    select = 2 * N * (S * H + H * I)                                   # DiscreteActor.forward
    reward = 2 * N * (I * H + S * H + H * H)                           # value_net(state, probs)
    grad = 2 * 2 * R * S * H + 2 * R * H * I * (3 + (n_chunks - 1) / n_chunks)
    return 3 * (select + reward + grad) + value_flops(S, H, H, I, N)


def make_agent(S, H, I, seed):
    torch.manual_seed(seed)
    with torch.device("cuda"):
        policy = recnn_b200.nn.DiscreteActor(S, I, H)
        value = recnn_b200.nn.Critic(S, I, H, 3e-3)
    agent = recnn_b200.nn.Reinforce(policy, value)
    agent.device = torch.device("cuda", torch.cuda.current_device())
    agent.optimizers["value_optimizer"] = recnn_b200.optim.Adam(agent.nets["value_net"].parameters(), lr=1e-4)
    agent.optimizers["policy_optimizer"] = recnn_b200.optim.Adam(agent.nets["policy_net"].parameters(), lr=1e-4)
    return agent


def make_batch(S, I, N, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return {"state": torch.randn(N, S, device="cuda", generator=g),
            "next_state": torch.randn(N, S, device="cuda", generator=g),
            "action": torch.randint(0, I, (N,), device="cuda", generator=g),
            "reward": torch.randint(1, 6, (N,), device="cuda", generator=g).float() - 3,
            "done": (torch.rand(N, device="cuda", generator=g) < 0.1).float()}


def one_hot(b, I):
    d = dict(b)
    d["action"] = torch.zeros(b["action"].shape[0], I, device="cuda")
    d["action"][torch.arange(b["action"].shape[0], device="cuda"), b["action"]] = 1
    return d


def timed(fn, warmup, repeats):
    """(times, peak): peak memory above the state before the first call, which allocates the call's workspace"""
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    fn()
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
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
    return times, peak


def record(name, S, H, I, N, times, peak, f, **extra):
    med = statistics.median(times)
    return {"config": name, "S": S, "H": H, "num_items": I, "rows": N, "chunk_items": RF._chunk_items(N, I),
            "time_s_median": med, "time_s_min": min(times), "time_s_max": max(times), "repeats": len(times),
            "flops": f, "tflops_per_s": f / med / 1e12, "share_of_tf32_datasheet": f / med / TF32_DATASHEET,
            "peak_extra_bytes": peak, "dense_action_bytes": N * I * 4, **extra}


def value_config(name, warmup, repeats):
    S, H, I, N = CONFIGS[name]
    agent = make_agent(S, H, I, 1)
    b = make_batch(S, I, N, 2)
    params = dict(agent.params)

    def call(batch=b, a=agent):
        return recnn_b200.nn.value_update(batch, params, a.nets, a.optimizers, a.device, {}, learn=True)

    call(make_batch(S, I, 8, 5))          # gradient and optimizer arenas exist before the measured call
    times, peak = timed(call, warmup, repeats)
    extra = {"mode": "item_ids", "loss": float(call())}
    if name == "A":
        # the same seeded nets and batch through both paths, one step each: loss and weight difference
        ids_agent, dense_agent = make_agent(S, H, I, 3), make_agent(S, H, I, 3)
        l_ids = float(call(b, ids_agent))
        l_dense = float(call(one_hot(b, I), dense_agent))
        diffs = []
        for p, q in zip(ids_agent.nets["value_net"].parameters(), dense_agent.nets["value_net"].parameters()):
            diffs.append(float((p - q).abs().max() / q.abs().max()))
        dense_b = one_hot(b, I)
        dense_times, dense_peak = timed(lambda: call(dense_b, dense_agent), warmup, repeats)
        extra.update(ids_vs_dense_loss_rel_diff=abs(l_ids - l_dense) / abs(l_dense),
                     ids_vs_dense_weights_max_rel_diff=max(diffs), dense_time_s_median=statistics.median(dense_times),
                     dense_peak_extra_bytes=dense_peak)
    res = record(name, S, H, I, N, times, peak, value_flops(S, H, H, I, N), **extra)
    del agent
    return res


def policy_step_config(warmup, repeats):
    S, H, I, N = CONFIGS["D"]
    agent = make_agent(S, H, I, 4)
    steps = agent.params["policy_step"]
    batches = [make_batch(S, I, N, 10 + i) for i in range(steps)]
    state = {"step": 0}

    def cycle_then_policy_step():
        # steps 1..9 of a cycle are untimed set-up (they save the rows); the timed call is the policy step
        out = None
        for i in range(1, steps + 1):
            agent._step = state["step"] * steps + i
            if i == steps:
                torch.cuda.synchronize()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                out = agent.update(batches[i - 1])
                e1.record()
                e1.synchronize()
                state["last"] = e0.elapsed_time(e1) / 1e3
            else:
                agent.update(batches[i - 1])
        state["step"] += 1
        assert out is not None
        return out

    times = []
    for _ in range(warmup):
        cycle_then_policy_step()
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    for _ in range(repeats):
        losses = cycle_then_policy_step()
        times.append(state["last"])
    peak = torch.cuda.max_memory_allocated() - base
    res = record("D", S, H, I, N, times, peak, policy_step_flops(S, H, I, N, steps), mode="reinforce_update_policy_step",
                 saved_rows=N * steps, losses=losses)
    del agent, batches
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--configs", default="A,B,C,D")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_reinforce_critic_vocab.py needs a GPU")
    result = {"metric": "reinforce_critic_vocab", **gpu_info(), "tf32_datasheet_flops": TF32_DATASHEET, "configs": []}
    for name in args.configs.split(","):
        res = policy_step_config(args.warmup, args.repeats) if name == "D" else value_config(name, args.warmup, args.repeats)
        result["configs"].append(res)
        print(json.dumps(res), file=sys.stderr, flush=True)
        gc.collect()
        torch.cuda.empty_cache()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
