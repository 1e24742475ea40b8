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

``recall_at_k`` compares an approximate search's ids (an IVF ``nprobe``) with the exact ones.

``slate_distances`` and ``slate_metrics`` describe served slates as sets (DESIGN.md, 4d-diversity).  ``ids`` is the
int64 [N, k] output of any serving call (``DiscreteActor.topk`` / ``sample_topk``, ``ItemIndex.search``,
``Critic.topk``), -1 marking an empty slot; a filled slot is an id >= 0.  With c_j the number of filled slots that
hold item j (the exposure counts, over all n_items items, zeros included):

  ild               mean over rows with >= 2 filled slots of the row's mean pairwise distance (intra-list diversity)
  ild_min           the same mean, of each row's smallest pairwise distance
  coverage          distinct recommended items / n_items
  gini              Gini index of c: sum_i (2i - n - 1) c_(i) / (n sum c), c sorted ascending, i from 1, n = n_items;
                    uniform exposure gives 0, all exposure on one item (n - 1) / n
  exposure_entropy  Shannon entropy, in bits, of c / sum c
  novelty           mean over filled slots of -log2((pop_j + 1) / (n_users + 1)), pop_j the number of users whose
                    history holds item j (``DeviceFrameFeed.item_popularity()``)
  rows, slots       rows and filled slots counted

Distances are scipy's ``cdist`` metrics between table rows: "euclidean" sqrt(sum_d (a_d - b_d)^2) and "cosine"
1 - a.b / (|a| |b|) clipped to [0, 2], except that a pair with a zero vector has cosine distance 1 (scipy: NaN).  They
are computed on the device from the resident table by one kernel (recnn_slate_distances), never through an
[N, k, dim] gather.
"""
from __future__ import annotations

import math
import numbers

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


def recall_at_k(approx_ids, exact_ids):
    """(per_row, mean): the recall of an approximate search against the exact one, e.g. ``ItemIndex.search`` with an
    IVF ``nprobe`` against a flat index or ``rank``.  approx_ids and exact_ids are int64 [n, k] (-1 pads an empty slot).
    per_row float64 [n] = |approx_r & exact_r| / |exact_r| over the filled slots (-1 ignored on both sides; NaN for a
    row whose exact slots are all empty); mean = the mean over the rows that are not NaN (NaN when there are none)."""
    a, e = torch.as_tensor(approx_ids), torch.as_tensor(exact_ids)
    for x, name in ((a, "approx_ids"), (e, "exact_ids")):
        if x.dim() != 2 or x.dtype.is_floating_point or x.dtype.is_complex or x.dtype == torch.bool:
            raise ValueError("%s must be a 2-D integer tensor [n, k] (got %s %s)" % (name, tuple(x.shape), x.dtype))
    if a.shape[0] != e.shape[0]:
        raise ValueError("approx_ids and exact_ids must have the same rows (got %d and %d)" % (a.shape[0], e.shape[0]))
    a = a.to(device=e.device, dtype=torch.int64)
    e = e.to(torch.int64)
    valid_e = e >= 0
    hit = ((e[:, :, None] == a[:, None, :]) & (a[:, None, :] >= 0)).any(2) & valid_e
    n_e = valid_e.sum(1).double()
    per_row = hit.sum(1).double() / n_e
    per_row[n_e == 0] = float("nan")
    ok = ~torch.isnan(per_row)
    mean = float(per_row[ok].mean()) if bool(ok.any()) else float("nan")
    return per_row, mean


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


_SLATE_METRICS = {"euclidean": 0, "cosine": 1}


def _slate_ids(ids):
    if not torch.is_tensor(ids) or ids.dim() != 2 or ids.dtype != torch.int64:
        raise ValueError("ids must be an int64 [N, k] tensor (got %s)"
                         % ("%s %s" % (tuple(ids.shape), ids.dtype) if torch.is_tensor(ids) else type(ids).__name__))
    if not 1 <= ids.shape[1] <= 64:
        raise ValueError("a slate holds 1 <= k <= 64 slots (got k = %d)" % ids.shape[1])
    return ids


def _slate_args(ids, table, metric):
    """The checks of a distance call, before any device work: (ids, table), both contiguous."""
    from .. import _lib
    ids = _slate_ids(ids)
    if metric not in _SLATE_METRICS:
        raise ValueError("metric must be one of %s (got %r)" % (sorted(_SLATE_METRICS), metric))
    if not torch.is_tensor(table) or table.dim() != 2 or table.dtype != torch.float32 or table.shape[0] < 1 \
            or not 1 <= table.shape[1] < 2 ** 31:
        raise ValueError("table must be a non-empty fp32 [n_items, dim] tensor")
    if ids.device != table.device:
        raise ValueError("ids and table must be on the same device (ids on %s, table on %s)" % (ids.device, table.device))
    if table.device.type != "cuda":
        raise _lib.RecnnError("slate_distances runs on CUDA only (the table is on %s)" % table.device)
    return ids.contiguous(), table.detach().contiguous()


def slate_distances(ids, table, metric="cosine", matrix=False):
    """Pairwise distances between the items of each slate, from the embedding table: ``(mean, min, count)`` or, with
    ``matrix=True``, ``(mean, min, count, matrix)``, on the table's device.  Over the unordered pairs of filled slots
    of row n: ``mean`` fp32 [N] their mean distance, ``min`` fp32 [N] the smallest (both NaN for a row with fewer than
    2 filled slots), ``count`` int32 [N] the filled slots; ``matrix`` fp32 [N, k, k] every distance, symmetric bit for
    bit, 0 on the diagonal of filled slots and NaN wherever an empty slot is involved.

    ``ids`` int64 [N, k], 1 <= k <= 64, -1 for an empty slot; ``table`` fp32 [n_items, dim] on a CUDA device, the
    ids on the same device; ``metric`` "cosine" or "euclidean" (module docstring).  A row's results depend only on
    its own ids, bit for bit.  Nothing but the outputs is allocated.  Refused with ValueError before any device work:
    malformed ids, k outside [1, 64], an unknown metric, a table that is not fp32 [n_items, dim], and ids on another
    device than the table.  An id outside [-1, n_items) raises IndexError (after the call's one read-back)."""
    from .. import _lib
    ids, table = _slate_args(ids, table, metric)
    n, k = ids.shape
    dev = table.device
    mean = torch.empty(n, dtype=torch.float32, device=dev)
    mn = torch.empty(n, dtype=torch.float32, device=dev)
    count = torch.empty(n, dtype=torch.int32, device=dev)
    mat = torch.empty(n, k, k, dtype=torch.float32, device=dev) if matrix else None
    flag = torch.empty(1, dtype=torch.int32, device=dev)
    with torch.cuda.device(dev):
        _lib.check(_lib.lib().recnn_slate_distances(
            ids.data_ptr(), n, k, table.data_ptr(), table.shape[0], table.shape[1], _SLATE_METRICS[metric],
            mean.data_ptr(), mn.data_ptr(), count.data_ptr(), _lib.ptr(mat), flag.data_ptr(), _lib.stream_ptr(dev)))
    if int(flag.item()) != 0:
        raise IndexError("a slate id is outside [-1, %d)" % table.shape[0])
    return (mean, mn, count, mat) if matrix else (mean, mn, count)


def slate_metrics(ids, table=None, n_items=None, metric="cosine", popularity=None, n_users=None, group=None):
    """Diversity, coverage, exposure concentration and novelty of served slates ``ids`` int64 [N, k] (-1: empty slot),
    as a dict of floats with the definitions of the module docstring.  ``table`` (fp32 [n_items, dim], the ids'
    device) adds ``ild`` and ``ild_min`` under ``metric`` (``slate_distances``); ``n_items`` defaults to the table's or
    the popularity's length; ``popularity`` (integer counts [n_items], e.g. ``DeviceFrameFeed.item_popularity()``) with
    ``n_users`` (e.g. ``feed.csr.n_users``) adds ``novelty``.  A mean over nothing is NaN.

    ``group``: a torch.distributed process group; the exposure counts and the sums are all-reduced first, so
    data-parallel ranks that each hold their own rows report the global values.  The ids' device must suit the group's
    backend (CPU for gloo, CUDA for NCCL).  Refused with ValueError before any device work: what ``slate_distances``
    refuses, no ``n_items``, a popularity that is not an integer vector of n_items counts, and popularity without
    ``n_users``.  An id outside [-1, n_items) raises IndexError."""
    ids = _slate_ids(ids)
    if table is not None:
        ids, table = _slate_args(ids, table, metric)
        if n_items is None:
            n_items = int(table.shape[0])
        elif int(n_items) != table.shape[0]:
            raise ValueError("n_items = %d but the table has %d rows" % (n_items, table.shape[0]))
    if popularity is not None:
        popularity = torch.as_tensor(popularity)
        if popularity.dim() != 1 or popularity.dtype.is_floating_point or popularity.dtype == torch.bool \
                or popularity.dtype.is_complex:
            raise ValueError("popularity must be a 1-D integer tensor of counts")
        if n_items is None:
            n_items = int(popularity.shape[0])
        if popularity.shape[0] != n_items:
            raise ValueError("popularity holds %d counts for %d items" % (popularity.shape[0], n_items))
        if isinstance(n_users, bool) or not isinstance(n_users, numbers.Integral) or n_users < 0:
            raise ValueError("novelty needs n_users, an int >= 0 (got %r)" % (n_users,))
    if isinstance(n_items, bool) or not isinstance(n_items, numbers.Integral) or n_items < 1:
        raise ValueError("slate_metrics needs n_items >= 1 (or a table or popularity to take it from), got %r"
                         % (n_items,))
    n_items = int(n_items)
    dev = ids.device
    filled = ids[ids >= 0]
    if ids.numel() and (int(ids.min()) < -1 or (filled.numel() and int(filled.max()) >= n_items)):
        raise IndexError("a slate id is outside [-1, %d)" % n_items)
    counts = torch.bincount(filled, minlength=n_items)
    f64 = lambda x: torch.as_tensor(x, dtype=torch.float64, device=dev).reshape(())
    parts = [f64(ids.shape[0]), f64(filled.numel())]
    if table is not None:
        mean, mn, count = slate_distances(ids, table, metric)
        ok = count >= 2
        parts += [mean[ok].double().sum(), mn[ok].double().sum(), ok.sum().double()]
    if popularity is not None:
        pop = popularity.to(device=dev, dtype=torch.float64)[filled]
        parts.append((math.log2(n_users + 1.0) - torch.log2(pop + 1.0)).sum())
    sums = torch.stack(parts)
    if group is not None:
        import torch.distributed as dist
        dist.all_reduce(counts, group=group)
        dist.all_reduce(sums, group=group)
    s = sums.tolist()
    nan = float("nan")
    c = counts.double()
    total = float(c.sum())
    out = {"coverage": float((counts > 0).sum()) / n_items}
    if total > 0:
        ranks = torch.arange(1, n_items + 1, dtype=torch.float64, device=dev)
        out["gini"] = float(((2 * ranks - n_items - 1) * torch.sort(c).values).sum()) / (n_items * total)
        p = c[c > 0] / total
        out["exposure_entropy"] = float(-(p * torch.log2(p)).sum())
    else:
        out["gini"] = out["exposure_entropy"] = nan
    if table is not None:
        out["ild"] = s[2] / s[4] if s[4] else nan
        out["ild_min"] = s[3] / s[4] if s[4] else nan
    if popularity is not None:
        out["novelty"] = s[-1] / s[1] if s[1] else nan
    out["rows"] = int(s[0])
    out["slots"] = int(s[1])
    return out
