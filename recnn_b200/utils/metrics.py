"""Offline evaluation: ranking metrics from exact ranks, and importance-weighted estimates of a policy's reward.

Ranking metrics come from exact ranks (``DiscreteActor.rank``, ``ItemIndex.rank``): rank r of a held-out item is
the number of eligible items recommended before it, so r = 0 is the first slot.

  hit@k   mean of [r < k]
  NDCG@k  mean of [r < k] / log2(r + 2)      (one relevant item per row: the ideal DCG is 1)
  MRR     mean of 1 / (r + 1)                (over the whole list: no cut-off)

Pure torch on the ranks' device; ``ranking_metrics(..., group=)`` all-reduces the sums and the row count over a
``torch.distributed`` process group, so data-parallel ranks that each hold their own rows report the global means.

``off_policy_estimates`` estimates the reward the policy pi would earn from logged rows (s, a, r) of the behaviour
policy beta, with the Top-K off-policy correction's importance weights (DESIGN.md, 4d-ope).
"""
from __future__ import annotations

import math

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


def _real_rows(x, name):
    t = torch.as_tensor(x)
    if t.dim() != 1 or not (t.dtype.is_floating_point or t.dtype in (torch.int32, torch.int64)):
        raise ValueError("%s must be a 1-D real tensor (got %s %s)" % (name, tuple(t.shape), t.dtype))
    t = t.to(torch.float64)
    if not bool(torch.isfinite(t).all()):
        raise ValueError("%s holds a non-finite value" % name)
    return t


def off_policy_estimates(pi_log_prob, beta_log_prob, reward, K=1, clip=None, group=None):
    """Importance-weighted estimates of the reward the policy pi would earn, from N logged rows (s_n, a_n, r_n) of a
    behaviour policy beta: ``pi_log_prob`` = log pi(a_n | s_n) (``DiscreteActor.log_prob``), ``beta_log_prob`` =
    log beta(a_n | s_n) (``Beta.log_prob``, or logged propensities), ``reward`` r_n, each a 1-D tensor of N values.

    Row n's weight is w_n = alpha_K / beta with alpha_K = 1 - (1 - pi)^K, the probability that a slate of K items
    drawn with replacement from pi contains a_n (the Top-K correction's weight; K = 1 gives pi / beta).  It is formed
    in logs, log alpha_K = log(-expm1(K log1p(-pi))), so it stays exact at K = 1 and accurate for pi ~ 1e-7.  Returns
    a dict of floats (float64 arithmetic):

      ips            mean of w r                       (inverse propensity scoring; unbiased when beta > 0 on pi's support)
      snips          sum w r / sum w                   (self-normalised IPS: biased, lower variance)
      ess            (sum w)^2 / sum w^2               (effective sample size, n when every weight is equal)
      ips_stderr     standard error of ips            (sample standard deviation of w r over sqrt(n))
      max_weight     max w
      logged_reward  mean of r                         (the behaviour policy's own reward)
      n              rows
      clipped_ips    mean of min(w, clip) r            (with ``clip``)
      clipped_share  share of rows with w > clip       (with ``clip``)

    ``group``: a torch.distributed process group; the sums are all-reduced (and the maximum weight max-reduced) first,
    so data-parallel ranks that each hold their own rows report the global values.  The tensors' device must suit the
    group's backend (CPU for gloo, CUDA for NCCL).  Refused with ValueError: mismatched shapes, K not an int >= 1,
    clip <= 0 and a non-finite log-probability or reward."""
    lp_pi = _real_rows(pi_log_prob, "pi_log_prob")
    lp_beta = _real_rows(beta_log_prob, "beta_log_prob").to(lp_pi.device)
    r = _real_rows(reward, "reward").to(lp_pi.device)
    if not lp_pi.shape == lp_beta.shape == r.shape:
        raise ValueError("pi_log_prob, beta_log_prob and reward must have the same shape (got %s, %s, %s)"
                         % (tuple(lp_pi.shape), tuple(lp_beta.shape), tuple(r.shape)))
    if isinstance(K, bool) or not isinstance(K, int) or K < 1:
        raise ValueError("K must be an int >= 1, got %r" % (K,))
    if clip is not None and (isinstance(clip, bool) or not isinstance(clip, (int, float)) or not clip > 0):
        raise ValueError("clip must be None or a number > 0, got %r" % (clip,))
    lp_pi = lp_pi.clamp(max=0.0)                 # an fp32 log-prob can round a hair above 0; pi <= 1
    if K == 1:
        log_alpha = lp_pi
    else:
        pi = torch.exp(lp_pi)
        # alpha_K = K pi to first order: the form for a pi that underflows float64
        log_alpha = torch.where(pi > 0, torch.log(-torch.expm1(K * torch.log1p(-pi))), lp_pi + math.log(K))
    w = torch.exp(log_alpha - lp_beta)
    wr = w * r
    parts = [wr.sum(), w.sum(), (w * w).sum(), (wr * wr).sum(), r.sum(),
             torch.tensor(float(r.numel()), dtype=torch.float64, device=r.device)]
    if clip is not None:
        parts += [(torch.clamp(w, max=float(clip)) * r).sum(), (w > clip).double().sum()]
    sums = torch.stack(parts)
    top = (w.max() if w.numel() else torch.tensor(0.0, dtype=torch.float64, device=w.device)).reshape(1)
    if group is not None:
        import torch.distributed as dist
        dist.all_reduce(sums, group=group)
        dist.all_reduce(top, op=dist.ReduceOp.MAX, group=group)
    s = sums.tolist()
    n = int(s[5])
    nan = float("nan")
    ips = s[0] / n if n else nan
    out = {"ips": ips,
           "snips": s[0] / s[1] if n and s[1] > 0 else nan,
           "ess": s[1] * s[1] / s[2] if n and s[2] > 0 else nan,
           "ips_stderr": math.sqrt(max(s[3] - n * ips * ips, 0.0) / (n - 1) / n) if n > 1 else nan,
           "max_weight": float(top) if n else nan,
           "logged_reward": s[4] / n if n else nan,
           "n": n}
    if clip is not None:
        out["clipped_ips"] = s[6] / n if n else nan
        out["clipped_share"] = s[7] / n if n else nan
    return out
