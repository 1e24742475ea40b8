"""Item-set tables: the items each row of a serving call must not return, e.g. everything a user has already rated.

A table is ``ids int64[T]`` plus ``offsets int64[n_sets + 1]``: set s is ``ids[offsets[s]:offsets[s + 1]]``, sorted
ascending.  ``DiscreteActor.topk`` and ``ItemIndex.search`` take one as ``exclude=`` with an optional
``exclude_rows=`` (int64 [N]: the set of each row, -1 for none), so the rows of many windows of one user share that
user's set instead of each carrying a copy.  ``DeviceFrameFeed.seen_items()`` builds the table of the resident
histories.

The ids are checked against the vocabulary on the device when a call reads them, and only for the sets its rows
reference: an id outside ``[0, num_items)`` raises ``IndexError``; a set that is not ascending, or an
``exclude_rows`` value outside ``[-1, n_sets)``, raises ``ValueError``.
"""
from __future__ import annotations

import torch

_INT = (torch.int64, torch.int32, torch.int16, torch.int8, torch.uint8)


def _int_vector(x, name):
    t = torch.as_tensor(x)
    if t.dim() != 1 or t.dtype not in _INT:
        raise ValueError("%s must be a 1-D integer tensor (got %s %s)" % (name, tuple(t.shape), t.dtype))
    return t.to(torch.int64)


class ItemSets:
    """``ItemSets(ids, offsets, unique=False, device=None)``: sorts every set ascending (and drops repeated ids with
    ``unique=True``) once, on ``device`` (default: the ids' device).  ``offsets`` must start at 0, end at
    ``len(ids)`` and never decrease."""

    def __init__(self, ids, offsets, unique=False, device=None):
        ids, offsets = _int_vector(ids, "ids"), _int_vector(offsets, "offsets")
        device = ids.device if device is None else torch.device(device)
        n = offsets.numel() - 1
        if n < 0:
            raise ValueError("offsets needs n_sets + 1 >= 1 entries")
        off_h = offsets.cpu()
        if int(off_h[0]) != 0 or int(off_h[-1]) != ids.numel() or bool((off_h[1:] < off_h[:-1]).any()):
            raise ValueError("offsets must start at 0, end at len(ids) = %d and never decrease" % ids.numel())
        ids, offsets = ids.to(device), offsets.to(device)
        lengths = offsets[1:] - offsets[:-1]
        seg = torch.repeat_interleave(torch.arange(n, device=device), lengths)
        order = torch.argsort(ids, stable=True)
        order = order[torch.argsort(seg[order], stable=True)]         # by set, then by id
        ids = ids[order]
        if unique and ids.numel():
            keep = torch.ones_like(ids, dtype=torch.bool)
            keep[1:] = (ids[1:] != ids[:-1]) | (seg[1:] != seg[:-1])
            ids = ids[keep]
            lengths = torch.bincount(seg[keep], minlength=n)
            offsets = torch.zeros(n + 1, dtype=torch.int64, device=device)
            torch.cumsum(lengths, 0, out=offsets[1:])
        self.ids, self.offsets = ids.contiguous(), offsets.contiguous()

    @classmethod
    def from_lists(cls, lists, unique=False, device=None):
        """One set per list of item ids (any order)."""
        lists = [torch.as_tensor(x, dtype=torch.int64).reshape(-1) for x in lists]
        offsets = torch.zeros(len(lists) + 1, dtype=torch.int64)
        torch.cumsum(torch.tensor([x.numel() for x in lists], dtype=torch.int64), 0, out=offsets[1:])
        ids = torch.cat(lists) if lists else torch.zeros(0, dtype=torch.int64)
        return cls(ids, offsets, unique=unique, device=device)

    def __len__(self):
        return self.offsets.numel() - 1

    @property
    def device(self):
        return self.ids.device

    def to(self, device):
        """The same table on ``device`` (self when it is already there)."""
        device = torch.device(device)
        if self.ids.device == device:
            return self
        out = ItemSets.__new__(ItemSets)
        out.ids, out.offsets = self.ids.to(device), self.offsets.to(device)
        return out

    def set(self, s):
        """The ids of set s (ascending)."""
        return self.ids[int(self.offsets[s]):int(self.offsets[s + 1])]


def row_map(sets, exclude_rows, n):
    """(sets, row_set) for a call over n rows, with the refusals that need no device: ``exclude_rows`` None maps row
    r to set r and needs ``len(sets) == n``."""
    if exclude_rows is None:
        if len(sets) != n:
            raise ValueError("exclude has %d sets but the call has %d rows; pass exclude_rows to map rows to sets"
                             % (len(sets), n))
        return sets, None
    rows = _int_vector(exclude_rows, "exclude_rows")
    if rows.numel() != n:
        raise ValueError("exclude_rows must have one entry per row (%d), got %d" % (n, rows.numel()))
    return sets, rows
