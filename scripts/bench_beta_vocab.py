"""One call of the Top-K notebook's behaviour policy (nn.Beta: forward, loss, backward, RAdam step) at the notebook's
shapes and at a million items, next to an eager fp32 PyTorch Beta of the same shape (torch.optim.RAdam in place of
torch_optimizer's), reporting OOM where the eager class does not fit.

    python scripts/bench_beta_vocab.py [--out results.json]

Per shape: the median of 3 CUDA-event timings after a warm-up call; the algorithmic TFLOP/s (two GEMMs of 2 N S num_items
flops each: the logits and dW) and the share of the data-sheet dense TF32 rate that the native call's tensor-core work
amounts to (3xTF32 issues three MMA passes per product, so the share is 3 x algorithmic / peak; for the eager cuBLAS
SGEMM it is reported on the same footing for comparison only); the peak memory of the first call above the resident
model, and in all.  Every (shape, implementation) pair runs in a process of its own, so that nothing of an earlier
measurement is on the device.  The card's name and power limit are read, not set."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import recnn_b200  # noqa: E402

TF32_PEAK = 495e12           # H100 SXM data sheet, dense TF32
SHAPES = [(1290, 5000, 10), (1290, 5000, 2048), (1290, 1 << 20, 2048), (2570, 1 << 20, 2048)]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name()


class EagerBeta(torch.nn.Module):
    """The notebook's cell 3 with the shape as arguments and torch.optim.RAdam(decoupled_weight_decay=True)."""

    def __init__(self, S, items):
        super().__init__()
        self.net = torch.nn.Sequential(torch.nn.Linear(S, items), torch.nn.Softmax(dim=1))
        self.optim = torch.optim.RAdam(self.net.parameters(), lr=1e-5, weight_decay=1e-5, decoupled_weight_decay=True)
        self.criterion = torch.nn.CrossEntropyLoss()

    def forward(self, state, action):
        predicted_action = self.net(state)
        loss = self.criterion(predicted_action, action.argmax(1))
        self.optim.zero_grad()
        loss.backward()
        self.optim.step()
        return predicted_action.detach()


def time_calls(fn, reps=3):
    times = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b) / 1e3)
    return sorted(times)[len(times) // 2]


def run(kind, S, items, n):
    torch.manual_seed(0)
    dev = torch.device("cuda")
    try:
        with torch.device(dev):
            beta = recnn_b200.nn.Beta(S, items) if kind == "native" else EagerBeta(S, items)
        state = torch.randn(n, S, device=dev)
        ids = torch.randint(0, items, (n,), device=dev)
        # the notebook's batch is one-hot; the native call also takes the ids (nothing [N, num_items] besides probs)
        action = ids if kind == "native" else torch.nn.functional.one_hot(ids, items).float()
        if kind == "native":
            beta.optim.c_net(beta)                           # the moment arenas exist before the measurement
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        beta(state, action)
        torch.cuda.synchronize()
        peak = torch.cuda.max_memory_allocated() - base
        total = torch.cuda.max_memory_allocated()
        t = time_calls(lambda: beta(state, action))
    except torch.OutOfMemoryError:
        return {"kind": kind, "oom": True}
    flops = 2 * 2.0 * n * S * items
    return {"kind": kind, "seconds": t, "tflops": flops / t / 1e12, "tf32_share": 3 * flops / t / TF32_PEAK,
            "peak_first_call_gb": peak / 1e9, "peak_total_gb": total / 1e9}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--one", nargs=4, metavar=("KIND", "S", "ITEMS", "ROWS"), default=None,
                    help="measure one (implementation, shape) in this process and print its JSON line")
    args = ap.parse_args()
    if args.one:
        kind, S, items, n = args.one[0], *map(int, args.one[1:])
        print(json.dumps(dict(run(kind, S, items, n), S=S, num_items=items, rows=n)))
        return
    res = {"card": card(), "rows": []}
    print(res["card"])
    for S, items, n in SHAPES:
        for kind in ("native", "eager"):
            p = subprocess.run([sys.executable, os.path.abspath(__file__), "--one", kind, str(S), str(items), str(n)],
                               capture_output=True, text=True)
            if p.returncode != 0:
                raise RuntimeError("measurement %s %d/%d/%d failed:\n%s" % (kind, S, items, n, p.stderr[-2000:]))
            r = json.loads(p.stdout.strip().splitlines()[-1])
            res["rows"].append(r)
            print(json.dumps(r))
            sys.stdout.flush()
    if args.out:
        with open(args.out, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
