"""Off-policy estimation: the log-probs of logged items under the REINFORCE policy (DiscreteActor.log_prob) and the
behaviour policy (Beta.log_prob), against the calls they replace -- DiscreteActor.rank (whose pass 1 log_prob is) and
Beta.forward (the only way to get beta's probabilities before this, a training step with a dense output).

Prints one JSON line.  S 2570 / H 256 / 2^20 items; rows 2,048 and 16,384 for the policy, 2,048 for beta (Beta.forward
needs an [N, 2^20] output, which does not fit at 16,384 rows).  "rank_share": one rank's log_prob at W = 8 (its 131,072
items) through the public modules, with the all-gather replaced by a local copy of the record (the other ranks' records
are copies of this one's, headers fixed up): a per-rank compute time, not an 8-GPU measurement.  Action ids are uniform.

Per case: the median / min / max CUDA-event time of one call over --repeats calls after --warmup calls and the peak
torch.cuda.max_memory_allocated() above the inputs during one call (bench_recommend.timed); each log_prob case carries
its time ratio to the call it replaces on the same inputs.  The card's name, power limit and maximum SM clock are read
in the same run.
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
from recnn_b200 import _lib  # noqa: E402
from recnn_b200 import dist as D  # noqa: E402
from recnn_b200.nn.arena import param_arena  # noqa: E402
from bench_recommend import gpu_info, timed  # noqa: E402

S, H, ITEMS = 2570, 256, 1 << 20
ROWS = (2048, 16384)
BETA_ROWS = 2048
WORLD = 8


def free():
    gc.collect()
    torch.cuda.empty_cache()


def inputs(n, items=ITEMS):
    g = torch.Generator(device="cuda").manual_seed(n)
    return torch.randn(n, S, device="cuda", generator=g), torch.randint(0, items, (n,), device="cuda", generator=g)


class LocalGather:
    """A rank's communicator whose all-gather is a local copy: W copies of the rank's record with the headers of the
    W-rank plan, so the finish sees a valid plan."""
    capacity = 1 << 62

    def __init__(self, world, items):
        self.plan = torch.tensor([D.vocab_shard(items, q, world) for q in range(world)], dtype=torch.int32,
                                 device="cuda")
        self.world = world

    def all_gather(self, t):
        g = t.reshape(1, -1).repeat(self.world, 1)
        g[:, :2].view(torch.int32).copy_(self.plan)
        return g.reshape(-1)

    def close(self):
        pass


def rank_share_vp(world):
    rank = world - 1
    lo, hi = D.vocab_shard(ITEMS, rank, world)
    return D.VocabParallel(lo, hi, ITEMS, None, rank, world, LocalGather(world, ITEMS)), hi - lo


def policy_cases(warmup, repeats):
    torch.manual_seed(1)
    with torch.device("cuda"):
        m = recnn_b200.nn.DiscreteActor(S, ITEMS, H)
    param_arena(m)
    out = []
    for n in ROWS:
        state, action = inputs(n)
        res = {"rows": n, "num_items": ITEMS}
        res["rank"] = timed(lambda: m.rank(state, action), warmup, repeats)
        res["log_prob"] = timed(lambda: m.log_prob(state, action), warmup, repeats)
        res["log_prob"]["time_ratio_to_rank"] = res["log_prob"]["time_s_median"] / res["rank"]["time_s_median"]
        out.append(res)
        del state, action
        free()
    del m
    free()
    return out


def policy_rank_share(warmup, repeats):
    vp, local = rank_share_vp(WORLD)
    torch.manual_seed(1)
    with torch.device("cuda"):
        m = recnn_b200.nn.DiscreteActor(S, local, H)
    m.__dict__["_recnn_vp"] = vp
    param_arena(m)
    out = []
    for n in ROWS:
        state, action = inputs(n)
        res = {"rows": n, "world": WORLD, "rank": vp.rank, "local_items": local}
        res["log_prob"] = timed(lambda: m.log_prob(state, action), warmup, repeats)
        out.append(res)
        del state, action
        free()
    del m
    free()
    return out


def beta_cases(warmup, repeats):
    n = BETA_ROWS
    torch.manual_seed(2)
    with torch.device("cuda"):
        beta = recnn_b200.nn.Beta(S, ITEMS)
    beta.optim.c_net(beta)                              # the moment arenas exist before any measurement
    state, action = inputs(n)
    res = {"rows": n, "num_items": ITEMS}
    res["forward"] = timed(lambda: beta(state, action), warmup, repeats)
    res["log_prob"] = timed(lambda: beta.log_prob(state, action), warmup, repeats)
    res["log_prob"]["time_ratio_to_forward"] = res["log_prob"]["time_s_median"] / res["forward"]["time_s_median"]
    del beta
    free()
    vp, local = rank_share_vp(WORLD)
    torch.manual_seed(2)
    with torch.device("cuda"):
        shard = recnn_b200.nn.Beta(S, local)
    shard.__dict__["_recnn_vp"] = vp
    param_arena(shard)
    share = {"rows": n, "world": WORLD, "rank": vp.rank, "local_items": local}
    share["log_prob"] = timed(lambda: shard.log_prob(state, action), warmup, repeats)
    del shard, state, action
    free()
    return res, share


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--repeats", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_ope.py needs a GPU")
    result = {"metric": "off_policy_log_prob", **gpu_info(), "S": S, "H": H}
    result["policy"] = policy_cases(args.warmup, args.repeats)
    result["policy_rank_share"] = policy_rank_share(args.warmup, args.repeats)
    result["beta"], result["beta_rank_share"] = beta_cases(args.warmup, args.repeats)
    result["rank_share_note"] = ("one rank's compute with the all-gather replaced by a local copy; not an 8-GPU "
                                 "measurement")
    print(json.dumps(result))


if __name__ == "__main__":
    main()
