"""Offline ranking metrics from exact ranks (``DiscreteActor.rank``, ``ItemIndex.rank``): rank r of a held-out item is
the number of eligible items recommended before it, so r = 0 is the first slot.

  hit@k   mean of [r < k]
  NDCG@k  mean of [r < k] / log2(r + 2)      (one relevant item per row: the ideal DCG is 1)
  MRR     mean of 1 / (r + 1)                (over the whole list: no cut-off)

Pure torch on the ranks' device; ``ranking_metrics(..., group=)`` all-reduces the sums and the row count over a
``torch.distributed`` process group, so data-parallel ranks that each hold their own rows report the global means.
"""
from __future__ import annotations

import torch


def _ranks(ranks):
    r = torch.as_tensor(ranks)
    if r.dim() != 1 or r.dtype.is_floating_point or r.dtype.is_complex or r.dtype == torch.bool:
        raise ValueError("ranks must be a 1-D integer tensor (got %s %s)" % (tuple(r.shape), r.dtype))
    if r.numel() and int(r.min()) < 0:
        raise ValueError("ranks must be >= 0 (a rank of -1 marks a target outside the vocabulary)")
    return r.to(torch.float64)


def _k(k):
    if isinstance(k, bool) or not isinstance(k, int) or k < 1:
        raise ValueError("k must be a positive int, got %r" % (k,))
    return k


def _sums(r, ks):
    """float64 [2 * len(ks) + 1]: the hit and NDCG sums at each k, then the reciprocal-rank sum."""
    parts = []
    for k in ks:
        hit = r < k
        parts += [hit.double().sum(), torch.where(hit, 1.0 / torch.log2(r + 2.0), torch.zeros_like(r)).sum()]
    parts.append((1.0 / (r + 1.0)).sum())
    return torch.stack(parts)


def hit_rate(ranks, k):
    """Share of rows whose item is in the top k."""
    r = _ranks(ranks)
    return float((r < _k(k)).double().mean()) if r.numel() else float("nan")


def ndcg(ranks, k):
    """Mean NDCG@k with one relevant item per row."""
    r = _ranks(ranks)
    return float(_sums(r, (_k(k),))[1] / r.numel()) if r.numel() else float("nan")


def mrr(ranks):
    """Mean reciprocal rank."""
    r = _ranks(ranks)
    return float((1.0 / (r + 1.0)).mean()) if r.numel() else float("nan")


def ranking_metrics(ranks, ks=(1, 5, 10, 20), group=None):
    """``{"hit@k": ..., "ndcg@k": ... for k in ks, "mrr": ..., "n": rows}``.  With ``group`` (a torch.distributed
    process group, or ``torch.distributed.group.WORLD``) the sums and the row count are all-reduced first: every
    rank returns the means over all ranks' rows.  The ranks' device must suit the group's backend (CPU for gloo,
    CUDA for NCCL)."""
    ks = tuple(_k(k) for k in ks)
    r = _ranks(ranks)
    sums = torch.cat([_sums(r, ks), torch.tensor([float(r.numel())], dtype=torch.float64, device=r.device)])
    if group is not None:
        import torch.distributed as dist
        dist.all_reduce(sums, group=group)
    sums = sums.tolist()
    n = int(sums[-1])
    mean = (lambda s: s / n) if n else (lambda s: float("nan"))
    out = {}
    for i, k in enumerate(ks):
        out["hit@%d" % k] = mean(sums[2 * i])
        out["ndcg@%d" % k] = mean(sums[2 * i + 1])
    out["mrr"] = mean(sums[2 * len(ks)])
    out["n"] = n
    return out
