"""Serving slates sampled from the REINFORCE policy at a million-item vocabulary: DiscreteActor.sample_topk
(recnn_discrete_sample_topk[_sets]) against DiscreteActor.topk on the same rows, against forward + torch.multinomial
where the dense probabilities fit, and one rank's share of the vocabulary-parallel call.

Prints one JSON line.  Per case (S 2570 / H 256 / 1,000,000 items, k 10 and 64, rows 1, 128, 2,048 and 16,384, without
and with the long-tailed history sets of bench_recommend.py): the median / min / max CUDA-event time of one call over
--repeats calls after --warmup calls and the peak torch.cuda.max_memory_allocated() above the inputs during one call,
for sample_topk and topk, and their ratio.  Where the dense probabilities fit (rows <= 2,048), the same for forward +
torch.multinomial(replacement=False) (with sets: the rows' rated items zeroed first, on a dense mask made outside the
timing).

Pruning: an item is skipped without its Philox call and logs when logit + 16.75 (the bound of the noise) cannot beat
its thread's k-th key and the row's running k-th.  The kernel counts nothing, so the script reports, on the first 8
rows, the share of items whose bound is below the row's FINAL k-th perturbed key: an upper bound of what the pass
skips (the running k-th only reaches that value at the end).

The rank share: one rank of W = 8 (125,000 items) runs recnn_discrete_shard_sample_topk, the all-gather is replaced
by a local copy of its record with the other ranks' headers, then recnn_discrete_shard_sample_topk_finish.  It is one
GPU's compute, not an 8-GPU wall time.
"""
from __future__ import annotations

import argparse
import gc
import json
import os
import statistics
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from recnn_b200 import _lib  # noqa: E402
from recnn_b200 import dist as D  # noqa: E402
from recnn_b200.data import ItemSets  # noqa: E402
from recnn_b200.nn.arena import param_arena  # noqa: E402
from recnn_b200.nn.update import reinforce as RF  # noqa: E402
from scripts.bench_policy_topk import KS, ROWS, S, H, ITEMS, DENSE_MAX_ROWS, WORLD, gpu_info, policy, stats, \
    timed  # noqa: E402
from tests import _policy_sample_oracle as PS  # noqa: E402
from tests._philox import philox4x32_10  # noqa: E402

SEED = 12345
PRUNE_ROWS = 8


def history_sets(N, seed=144):
    """Long-tailed per-row sets as bench_recommend.py draws them (mean ~144 ids, a few >= 8,192)."""
    rng = np.random.default_rng(seed)
    lengths = np.minimum(rng.pareto(1.6, N) * 75 + 20, 20000).astype(np.int64)
    return [rng.integers(0, ITEMS, n) for n in lengths]


def prunable_share(m, state, ids, k):
    """The share of items of the first PRUNE_ROWS rows whose logit + G_max is below the row's final k-th key."""
    n = min(PRUNE_ROWS, state.shape[0])
    with torch.no_grad():
        h = torch.relu(state[:n] @ m.linear1.weight.T + m.linear1.bias)
        z = h @ m.linear2.weight.T + m.linear2.bias
    last = ids[:n, k - 1].clamp(min=0)
    zk = z.gather(1, last[:, None])[:, 0].double().cpu().numpy()
    hi = (np.arange(n, dtype=np.uint64) << np.uint64(8)) | np.uint64(PS.TAG)      # the k-th item's noise only
    x = philox4x32_10((last.cpu().numpy().astype(np.uint64), 0, hi & np.uint64(0xFFFFFFFF), hi >> np.uint64(32)),
                      (SEED & 0xFFFFFFFF, SEED >> 32))[0]
    g = -np.log(-np.log((2.0 * (x >> np.uint32(9)).astype(np.float64) + 1.0) * 2.0 ** -24))
    bar = torch.from_numpy(zk + g).to(z.device, torch.float32)
    return float((z + PS.G_MAX < bar[:, None]).double().mean())


def unsharded_cases(warmup, repeats):
    m = policy(ITEMS, 1)
    out = []
    for N in ROWS:
        state = torch.randn(N, S, device="cuda", generator=torch.Generator(device="cuda").manual_seed(N))
        lists = history_sets(N)
        for with_sets in (False, True):
            sets = ItemSets.from_lists(lists, device="cuda") if with_sets else None
            for k in KS:
                st, sp, (sv, si) = timed(lambda: m.sample_topk(state, k, exclude=sets, seed=SEED), warmup, repeats)
                tt, tp, _ = timed(lambda: m.topk(state, k, exclude=sets), warmup, repeats)
                res = {"rows": N, "k": k, "history_sets": with_sets, "num_items": ITEMS,
                       "chunk_items": RF._chunk_items(N, ITEMS),
                       "sample_topk": {**stats(st), "peak_bytes_during_call": sp},
                       "topk": {**stats(tt), "peak_bytes_during_call": tp},
                       "sample_over_topk": statistics.median(st) / statistics.median(tt),
                       "prunable_share_final_bar": prunable_share(m, state, si, k)}
                if N <= DENSE_MAX_ROWS:
                    keep = None
                    if with_sets:
                        keep = torch.ones(N, ITEMS, device="cuda")
                        rows = torch.cat([torch.full((len(x),), r, dtype=torch.int64) for r, x in enumerate(lists)])
                        keep[rows.cuda(), torch.from_numpy(np.concatenate(lists)).cuda()] = 0.0

                    def dense():
                        p = m(state)
                        if keep is not None:
                            p = p * keep
                        return torch.multinomial(p, k, replacement=False)
                    dt, dpeak, _ = timed(dense, warmup, repeats)
                    res["dense_multinomial"] = {**stats(dt), "peak_bytes_during_call": dpeak}
                    res["dense_over_sample"] = statistics.median(dt) / statistics.median(st)
                    del keep
                out.append(res)
                del sv, si
                gc.collect()
                torch.cuda.empty_cache()
            del sets
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
                rec = torch.empty(L.recnn_vocab_sample_topk_record_floats(N, k), device="cuda")
                _lib.check(L.recnn_discrete_shard_sample_topk(d, vs, param_arena(m).data_ptr(), state.data_ptr(), N,
                                                              k, None, 0, SEED, 0, chunk, rec.data_ptr(),
                                                              ws.data_ptr(), nbytes, st))
                del ws
                gathered = rec.repeat(WORLD)
                gathered.view(WORLD, -1)[:, :2].view(torch.int32).copy_(heads)
                values = torch.empty(N, k, device="cuda")
                ids = torch.empty(N, k, dtype=torch.int64, device="cuda")
                flag = torch.empty(1, dtype=torch.int32, device="cuda")
                _lib.check(L.recnn_discrete_shard_sample_topk_finish(d, vs, gathered.data_ptr(), N, k, None, 0, SEED,
                                                                     values.data_ptr(), ids.data_ptr(),
                                                                     flag.data_ptr(), st))
                return flag
            times, peak, flag = timed(call, warmup, repeats)
            out.append({"world": WORLD, "rank": rank, "local_items": hi - lo, "rows": N, "k": k, "chunk_items": chunk,
                        **stats(times), "peak_bytes_during_call": peak, "error_bits": int(flag.item()),
                        "note": "one rank's compute with the all-gather replaced by a local copy, not an 8-GPU time"})
        del state
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--repeats", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_policy_sample.py needs a GPU")
    result = {"metric": "policy_sample_topk", **gpu_info(), "S": S, "H": H}
    result["cases"] = unsharded_cases(args.warmup, args.repeats)
    result["rank_share"] = rank_share_cases(args.warmup, args.repeats)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
