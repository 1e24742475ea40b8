"""fp32 restatement of one Lloyd round of the device k-means (ivf_lloyd in csrc/ivf.cu, DESIGN.md 4c-ivf), given the
round's assignment.  The IVF coarse build and every IVF_PQ codebook run these rounds.

A device round is: an L2 assignment (recnn_retrieve_topk, k = 1), ivf_update_kernel, ivf_split_kernel and, for COS,
ivf_normalize_kernel.  The assignment goes through the GEMM, so the tests read it from the device or decide it here
only where float64 distances leave no doubt (decide()).  Given the assignment, the rest is IEEE arithmetic that numpy
reproduces bit for bit:

  update   each list's members in ascending point order, summed in float64 from +0.0, one add after another (not
           np.sum, which is pairwise); the sum divided by the count in float64, then rounded to float32.  An empty list
           keeps its centroid.
  split    float32 counts.  Empty lists in ascending id; the donor is the largest count, ties to the smaller id.  The
           empty list gets the donor's centroid with even dims * float32(1 + 2^-10) and odd dims * float32(1 - 2^-10),
           the donor the opposite; half = count[donor] * 0.5 goes to the empty list and count[donor] - half stays,
           both in float32, before the next donor is chosen.

The COS renormalisation sums squares in warp order with fmaf; it is held to a bound (see the COS test), not to bits."""
from __future__ import annotations

import numpy as np

U = 2.0 ** -24                        # fp32 unit roundoff
EPS = np.float32(1.0 / 1024.0)
UP = np.float32(1.0) + EPS            # both exact in float32
DOWN = np.float32(1.0) - EPS


def update(points, assign, centroids):
    """(centroids float32 [k, dim], counts float32 [k]): each non-empty list's mean as ivf_update_kernel computes it"""
    x = np.asarray(points, np.float32)
    c = np.array(centroids, np.float32, copy=True)
    assign = np.asarray(assign, np.int64)
    counts = np.bincount(assign, minlength=len(c))
    order = np.argsort(assign, kind="stable")          # each list's members, ascending
    offs = np.concatenate([[0], np.cumsum(counts)])
    zero = np.zeros((1, x.shape[1]), np.float64)
    for l in np.nonzero(counts)[0]:
        members = x[order[offs[l]:offs[l + 1]]].astype(np.float64)
        # sequential: each partial sum rounds once, as the kernel's `s += ...`; the leading +0.0 row makes a list of
        # -0.0 entries sum to +0.0, as the kernel's `double s = 0.0` does
        s = np.add.accumulate(np.concatenate([zero, members]), axis=0)[-1]
        c[l] = (s / np.float64(counts[l])).astype(np.float32)
    return c, counts.astype(np.float32)


def split(c, counts):
    """ivf_split_kernel in place on float32 c [k, dim] and counts [k]; returns the (empty, donor) pairs in order"""
    even = np.arange(c.shape[1]) % 2 == 0
    to_empty, to_donor = np.where(even, UP, DOWN), np.where(even, DOWN, UP)
    pairs = []
    for i in range(len(counts)):
        if counts[i] != 0:
            continue
        j = int(np.argmax(counts))                    # the first maximum: ties to the smaller id
        v = c[j].copy()
        c[i] = v * to_empty
        c[j] = v * to_donor
        half = counts[j] * np.float32(0.5)
        counts[i] = half
        counts[j] = counts[j] - half
        pairs.append((i, j))
    return pairs


def round_(points, assign, centroids):
    """one round without the COS renormalisation: (centroids float32, counts after the split, (empty, donor) pairs)"""
    c, counts = update(points, assign, centroids)
    pairs = split(c, counts)
    return c, counts, pairs


def sq_dists(points, c):
    """float64 [n, k] squared distances (|x|^2 + |c|^2 - 2 <x, c>: its own error is ~1e-16 of the terms, far below
    the fp32 bars it is compared with)"""
    x, c = np.asarray(points, np.float64), np.asarray(c, np.float64)
    return np.maximum((x * x).sum(1)[:, None] + (c * c).sum(1)[None, :] - 2.0 * (x @ c.T), 0.0)


def key_bar(points, c):
    """float64 [n]: how far apart the float64 distances of two centroids can be while the device ranks them the other
    way.  The device ranks key_j = |c_j|^2 - 2 <x, c_j> (|x|^2 is common to every key).  On either GEMM back end the
    product <x, c_j> of dim terms has an error of at most (dim + 1) * 2^-20 * sum_d |x_d c_jd|: a 3xTF32 product
    drops the lo * lo term and rounds the lo parts (< 3 * 2^-22 relative, below 2^-20), and each of the dim fp32
    accumulations rounds once (2^-24 relative to a partial sum bounded by the same sum).  |c_j|^2 has the same bound
    with |c_j|^2 in place of the sum, and the fma that forms the key rounds once more.  So
    |key_j - exact| <= (dim + 2) * 2^-20 * (|c_j|^2 + 2 |x| |c_j|) <= (dim + 2) * 2^-20 * (|x| + |c_j|)^2,
    and two keys compared: twice that, with the largest |c_j|."""
    x, c = np.asarray(points, np.float64), np.asarray(c, np.float64)
    dim = x.shape[1]
    cmax = np.sqrt((c * c).sum(1)).max()
    return 2.0 * (dim + 2) * 2.0 ** -20 * (np.sqrt((x * x).sum(1)) + cmax) ** 2


def gaps(points, c, assign):
    """float64 [n]: how much farther each point's assigned centroid is than its nearest one"""
    d = sq_dists(points, c)
    return d[np.arange(len(d)), np.asarray(assign, np.int64)] - d.min(1)


def candidates(points, c, bar):
    """bool [n, k]: the centroids within bar of each point's nearest"""
    d = sq_dists(points, c)
    return d <= d.min(1, keepdims=True) + np.asarray(bar, np.float64)[:, None]


def decide(points, c, bar):
    """(assign int64 [n], ambiguous bool [n]): the L2 assignment the device must make wherever it is decided.  The
    candidates of a point are the centroids within bar of its nearest.  Centroids with equal bits get equal keys on the
    device, and their tie goes to the smaller id; so when every candidate has the same bits the assignment is the
    smallest candidate id.  Otherwise the point is ambiguous."""
    c = np.asarray(c, np.float32)
    near = candidates(points, c, bar)
    first = np.argmax(near, axis=1)
    _, cls = np.unique(c.view(np.uint32), axis=0, return_inverse=True)   # one class per bit pattern
    cls = cls.reshape(-1)
    ambiguous = (near & (cls[None, :] != cls[first][:, None])).any(1)
    return first.astype(np.int64), ambiguous


def same_bits(a, b):
    return np.array_equal(np.asarray(a, np.float32).view(np.uint32), np.asarray(b, np.float32).view(np.uint32))
