"""REINFORCE policy gradient at large vocabularies: one recnn_reinforce_policy_grad_chunked call per timing, single chunk
vs the chunk width ChooseREINFORCE picks by itself (recnn_b200.nn.update.reinforce._chunk_items).

Prints one JSON line.  Per config: the median / min / max CUDA-event time of one call over --repeats calls after
--warmup calls, the peak torch.cuda.max_memory_allocated() above the inputs during one call (its scratch included), the
chunk width and count, and the scratch the single-chunk call would need (recnn_discrete_scratch_floats(d, R, 1)).

FLOPs are the algorithm's, counted from the shapes: 2 R S H for the layer-1 forward and again for dW1, plus 2 R H I for
each of the logits GEMM, dW2 and dh -- and once more for the logits of every chunk but the last when the items are
chunked (pass 2 recomputes them; the last chunk is still in the buffer) -- times 3 for the 3xTF32 passes on the tensor
cores.  The share of peak is against NVIDIA's data-sheet dense TF32 rate for the H100 SXM (495 TFLOP/s), a data-sheet
figure for a 700 W card, not a measured one.

Configs (S / H / num_items / R):
  A  1290 / 2048 / 5,000     / 1,280     the notebook shape, single chunk
  B  1290 / 2048 / 1,000,000 / 1,280     single chunk and auto-chunked: what the recompute costs
  C  2570 / 256  / 1,000,000 / 163,840   BASELINE configs[4]'s rows per policy update (16,384 x policy_step 10)
plus an informational line: DiscreteActor.forward + _sample for 1,280 rows at 1M items (H = 2048).
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
from recnn_b200.nn.arena import param_arena  # noqa: E402
from recnn_b200.nn.update import reinforce as RF  # noqa: E402

TF32_DATASHEET = 495e12
CONFIGS = {"A": (1290, 2048, 5_000, 1_280), "B": (1290, 2048, 1_000_000, 1_280), "C": (2570, 256, 1_000_000, 163_840)}


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, power, clock = (x.strip() for x in q.stdout.splitlines()[0].split(","))
    return {"gpu": name, "power_limit": power, "max_sm_clock": clock}


def flops(S, H, I, R, n_chunks):
    logit_gemms = 3 + (n_chunks - 1) / n_chunks
    return 3 * (2 * 2 * R * S * H + 2 * R * H * I * logit_gemms)


def make_inputs(S, H, I, R, seed):
    torch.manual_seed(seed)
    with torch.device("cuda"):
        m = recnn_b200.nn.DiscreteActor(S, I, H)
    g = torch.Generator(device="cuda").manual_seed(seed)
    state = torch.randn(R, S, device="cuda", generator=g)
    action = torch.randint(0, I, (R,), device="cuda", generator=g)
    blp = torch.log(torch.empty(R, device="cuda").uniform_(0.5 / I, 2.0 / I, generator=g))
    ret = torch.randn(R, device="cuda", generator=g)
    return m, state, action, blp, ret


def time_call(m, state, action, blp, ret, chunk, warmup, repeats):
    L = _lib.lib()
    d = m.dims
    R = state.shape[0]
    flat = param_arena(m)
    grads = torch.zeros_like(flat)
    out = torch.zeros(2, device="cuda")
    st = _lib.stream_ptr()

    def call(scratch):
        _lib.check(L.recnn_reinforce_policy_grad_chunked(d, flat.data_ptr(), grads.data_ptr(), state.data_ptr(),
                                                         action.data_ptr(), blp.data_ptr(), ret.data_ptr(), R,
                                                         _lib.REINFORCE_TOPK, 10, chunk, out.data_ptr(),
                                                         scratch.data_ptr(), st))

    # peak memory of one call, its scratch allocation included (collect first: a module freed by the cycle collector
    # in the middle of the measurement would lower the baseline)
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.max_memory_allocated()
    scratch = torch.empty(L.recnn_reinforce_scratch_floats(d, R, chunk), device="cuda")
    call(scratch)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    for _ in range(warmup):
        call(scratch)
    times = []
    for _ in range(repeats):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        call(scratch)
        e1.record()
        e1.synchronize()
        times.append(e0.elapsed_time(e1) / 1e3)
    finite = bool(torch.isfinite(out[:1]).all() and torch.isfinite(grads).all())
    del scratch
    return times, peak, finite, float(out[0]), grads


def run_config(name, chunk_mode, warmup, repeats, inputs):
    S, H, I, R = CONFIGS[name]
    m, state, action, blp, ret = inputs
    chunk = I if chunk_mode == "single" else RF._chunk_items(R, I)
    n_chunks = -(-I // chunk)
    times, peak, finite, loss, grads = time_call(m, state, action, blp, ret, chunk, warmup, repeats)
    med = statistics.median(times)
    f = flops(S, H, I, R, n_chunks)
    single = _lib.lib().recnn_discrete_scratch_floats(m.dims, R, 1) * 4
    res = {"config": name, "S": S, "H": H, "num_items": I, "rows": R, "chunk_items": chunk, "n_chunks": n_chunks,
           "time_s_median": med, "time_s_min": min(times), "time_s_max": max(times), "repeats": len(times),
           "flops": f, "tflops_per_s": f / med / 1e12, "share_of_tf32_datasheet": f / med / TF32_DATASHEET,
           "peak_bytes_during_call": peak, "single_chunk_scratch_bytes": single, "loss": loss, "finite": finite}
    return res, grads


def sample_line(warmup, repeats, m):
    """DiscreteActor.forward + _sample for 1,280 rows at this actor's vocabulary."""
    S = m.linear1.in_features
    state = torch.randn(1280, S, device="cuda")
    for _ in range(warmup):
        m._sample(m(state))
    times = []
    for _ in range(repeats):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        m._sample(m(state))
        e1.record()
        e1.synchronize()
        times.append(e0.elapsed_time(e1) / 1e3)
    return {"rows": 1280, "num_items": m.linear2.out_features, "hidden": m.linear1.out_features,
            "time_s_median": statistics.median(times), "time_s_min": min(times), "time_s_max": max(times)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--configs", default="A,B,C")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_reinforce_vocab.py needs a GPU")
    result = {"metric": "reinforce_policy_grad_vocab", **gpu_info(), "tf32_datasheet_flops": TF32_DATASHEET,
              "configs": []}
    for name in args.configs.split(","):
        S, H, I, R = CONFIGS[name]
        inputs = make_inputs(S, H, I, R, seed=len(result["configs"]) + 1)
        modes = ["single", "auto"] if name == "B" else ["auto"]
        grads = {}
        for mode in modes:
            res, grads[mode] = run_config(name, mode, args.warmup, args.repeats, inputs)
            res["mode"] = mode
            result["configs"].append(res)
        if len(grads) == 2:
            a, b = grads["auto"], grads["single"]
            result["B_auto_vs_single_max_rel_diff"] = float((a - b).abs().max() / b.abs().max())
            result["B_time_ratio_auto_over_single"] = result["configs"][-1]["time_s_median"] / result["configs"][-2]["time_s_median"]
            result["sample_1m_items"] = sample_line(args.warmup, args.repeats, inputs[0])
        del inputs, grads
        gc.collect()
        torch.cuda.empty_cache()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
