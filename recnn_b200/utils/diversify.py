"""Diversified re-ranking of served candidate pools (DESIGN.md, 4d-diversify).

Every serving call returns a scored pool of candidates per row; ``diversify`` re-ranks that pool into a slate that
trades relevance against redundancy, measured by the cosine similarity of the items' rows in the resident embedding
table:

  "mmr"  maximal marginal relevance (Carbonell & Goldstein, 1998): step t picks the eligible item i maximising
         weight * s_i - (1 - weight) * max_{j already picked} sim(i, j)   (no penalty at the first step)
  "dpp"  greedy MAP inference of the DPP L = Diag(q) S Diag(q), S_ij = (1 + sim_ij) / 2, q_i = exp(alpha s_i),
         alpha = weight / (2 (1 - weight)) (Chen, Zhang & Zhou, NeurIPS 2018): step t picks the item that most increases
         log det L_S, i.e. argmax 2 alpha s_i + log d_i^2 with d_i^2 the Schur complement of i in S; it stops when that
         d^2 falls below 1e-4 (the pool holds no direction the slate does not already span).  At weight 1 it orders
         by score.

sim(a, b) = a.b / (|a| |b|), clipped to [-1, 1], 0 with a zero vector: 1 - ``slate_distances(metric="cosine")``, so
re-ranking acts on the ``ild`` / ``ild_min`` that ``slate_metrics`` reports.  One kernel (recnn_slate_diversify) reads
each candidate's row once into shared memory and runs the k greedy steps there; nothing of size [N, m, dim] is formed.
"""
from __future__ import annotations

import numbers

import torch

_METHODS = {"mmr": 0, "dpp": 1}


def diversify(ids, scores, table, k, method="mmr", weight=0.5):
    """Re-rank each row's candidate pool into a diverse slate of k items: ``(ids, pos, gain)``, each [N, k] on the
    table's device, in selection order.  ``ids`` int64 are the picked items, ``pos`` int64 each pick's column in the
    pool (so ``scores.gather(1, pos)`` gives the picks' scores), ``gain`` fp32 the objective at selection (module
    docstring; for the DPP the increase of log det L_S).  A row with fewer than k eligible items, or a DPP that stops,
    ends in -1 / -1 / NaN.

    ``ids`` int64 [N, m] is each row's pool (1 <= m <= 256; -1 padding; a pool may repeat an id, e.g. the union of two
    calls' pools, but a slate never does), ``scores`` fp32 [N, m] its relevance, higher is better.  Pass:

      ``DiscreteActor.topk`` / ``sample_topk`` values (pi)   ->  ``values.log()``  (log pi)
      ``Critic.topk`` values                                  ->  the Q values as they are
      ``ItemIndex.search`` with metric "L2"                   ->  ``-result.dist()``  (minus the distance)
      ``ItemIndex.search`` with metric "IP" or "COS"          ->  ``result.dist()``   (the similarity)

    ``table`` fp32 [n_items, dim] (1 <= dim <= 1024), e.g. ``DeviceFrameFeed.table`` or ``ItemIndex.table``, on a CUDA
    device, with ids and scores on the same device.  ``k`` in [1, min(64, m)]; ``method`` "mmr" or "dpp"; ``weight``
    in [0, 1]: 1 ranks by relevance only, 0 by diversity only.  Ties go to the smaller id, then the smaller column.  A
    row's outputs depend only on its own ids, scores and the table, bit for bit.  Nothing but the outputs and a flag is
    allocated.

    Refused with ValueError before any device work: malformed shapes or dtypes, m outside [1, 256], dim outside
    [1, 1024], k outside [1, min(64, m)], an unknown method, a weight outside [0, 1], tensors on different devices.  A
    table off the GPU raises RecnnError.  After the call's one read-back, an id outside [-1, n_items) raises IndexError
    and a non-finite score of a filled slot ValueError."""
    from .. import _lib
    if not torch.is_tensor(ids) or ids.dim() != 2 or ids.dtype != torch.int64:
        raise ValueError("ids must be an int64 [N, m] tensor (got %s)"
                         % ("%s %s" % (tuple(ids.shape), ids.dtype) if torch.is_tensor(ids) else type(ids).__name__))
    if not torch.is_tensor(scores) or scores.dtype != torch.float32 or scores.shape != ids.shape:
        raise ValueError("scores must be an fp32 tensor of the ids' shape %s (got %s)" % (
            tuple(ids.shape), "%s %s" % (tuple(scores.shape), scores.dtype) if torch.is_tensor(scores)
            else type(scores).__name__))
    n, m = ids.shape
    if not 1 <= m <= 256:
        raise ValueError("a pool holds 1 <= m <= 256 candidates (got m = %d)" % m)
    if not torch.is_tensor(table) or table.dim() != 2 or table.dtype != torch.float32 or table.shape[0] < 1 \
            or not 1 <= table.shape[1] <= 1024:
        raise ValueError("table must be a non-empty fp32 [n_items, dim] tensor with 1 <= dim <= 1024")
    if isinstance(k, bool) or not isinstance(k, numbers.Integral) or not 1 <= k <= min(64, m):
        raise ValueError("k must be an int in [1, min(64, m) = %d], got %r" % (min(64, m), k))
    if method not in _METHODS:
        raise ValueError("method must be one of %s (got %r)" % (sorted(_METHODS), method))
    if isinstance(weight, bool) or not isinstance(weight, numbers.Real) or not 0.0 <= weight <= 1.0:
        raise ValueError("weight must be a number in [0, 1], got %r" % (weight,))
    if not ids.device == scores.device == table.device:
        raise ValueError("ids, scores and table must be on one device (got %s, %s, %s)"
                         % (ids.device, scores.device, table.device))
    if table.device.type != "cuda":
        raise _lib.RecnnError("diversify runs on CUDA only (the table is on %s)" % table.device)
    k = int(k)
    dev = table.device
    ids, scores, table = ids.contiguous(), scores.detach().contiguous(), table.detach().contiguous()
    out_ids = torch.empty(n, k, dtype=torch.int64, device=dev)
    out_pos = torch.empty(n, k, dtype=torch.int64, device=dev)
    gain = torch.empty(n, k, dtype=torch.float32, device=dev)
    flag = torch.empty(1, dtype=torch.int32, device=dev)
    with torch.cuda.device(dev):
        _lib.check(_lib.lib().recnn_slate_diversify(
            ids.data_ptr(), scores.data_ptr(), n, m, k, table.data_ptr(), table.shape[0], table.shape[1],
            _METHODS[method], float(weight), out_ids.data_ptr(), out_pos.data_ptr(), gain.data_ptr(), flag.data_ptr(),
            _lib.stream_ptr(dev)))
    f = int(flag.item())
    if f & 1:
        raise IndexError("a pool id is outside [-1, %d)" % table.shape[0])
    if f & 2:
        raise ValueError("a filled pool slot has a non-finite score")
    return out_ids, out_pos, gain
