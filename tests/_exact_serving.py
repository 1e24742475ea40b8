"""Bit-exact restatement of serving through the REINFORCE policy (``DiscreteActor.topk`` / ``sample_topk`` / ``rank``
/ ``log_prob``) and the DDPG / TD3 critic (``Critic.topk`` / ``Critic.rank``) for nets of small integers.

When every GEMM operand is an integer with |x| <= 2^11 (policy: the state, W1, the hidden layer h and W2; critic: the
state, the item table, W1, h1 and W2), its TF32 hi part is the value and its lo part 0, so the 3xTF32 tensor-core GEMM
multiplies exactly, as the CUDA-core fp32 FMAs do.  When, for every output of every layer, sum |a_i b_i| + |bias| <
2^24, every partial sum in any order is an integer below 2^24 and so exact in fp32.  That covers the critic's
u_r + v_j and its warp dot w3 . h2 + b3 too.  Under both conditions every logit and every Q is the float64 value, on
either back end, and the builders below assert both in float64.

Then the orders are known bit for bit: a candidate is (key, id), key = fminf(-z, FLT_MAX) (policy) or
fminf(-Q, FLT_MAX) (critic), smaller key first and equal keys the smaller id; NaN and -inf logits rank after every
finite one and still before any pad.  The ids are a stable argsort of the keys over the eligible items; a rank counts
the eligible j != t with (key_j, j) < (key_t, t), the target never excluded.

Probabilities go through __expf and a reduction, so only rows built for it are exact: when a row's logits are all
either M (c of them) or at most M - 128, every exp term is exactly 1 or 0 (e^-128 is below fp32's smallest
subnormal), so S = c and pi is fp32(1 / c) for the tied items and 0 for the others.  Every other value is checked
against float64 within ``pi_bar``."""
from __future__ import annotations

import math

import numpy as np
import torch

from tests._exact_retrieval import FLT_MAX, finite_key, small_ints  # noqa: F401

OPERAND = 2 ** 11          # |GEMM operand| that TF32 holds exactly
SUM = 2 ** 24              # |partial sum| that fp32 holds exactly
NUM_SMS = 132              # H100 SXM: topk.cuh kNumSMs
TOPK_THREADS = 256
SPLIT_CAP = 31


# ----------------------------------------------------------------------------- builders
def _layer(x, w, b, what):
    """float64 x @ w.T + b after asserting that the layer is exact in fp32 on both back ends; non-finite biases (the
    masking tests) are added after the bound, which they do not affect"""
    x, w, b = np.asarray(x, np.float64), np.asarray(w, np.float64), np.asarray(b, np.float64)
    for t, name in ((x, "input"), (w, "weight")):
        assert np.all(np.isfinite(t)) and np.all(t == np.round(t)), "%s %s is not integer" % (what, name)
        assert np.abs(t).max(initial=0) <= OPERAND, "%s %s exceeds 2^11" % (what, name)
    fb = np.where(np.isfinite(b), b, 0.0)
    assert np.all(fb == np.round(fb)), "%s bias is not integer" % what
    bound = np.abs(x) @ np.abs(w).T + np.abs(fb)
    assert bound.max(initial=0) < SUM, "%s: a partial sum can reach 2^24 (%d)" % (what, bound.max())
    return x @ w.T + b


def _sparse_ints(rng, shape, nnz, lo, hi):
    """integers in [lo, hi] with nnz nonzero-candidates per row (the rest 0)"""
    out = np.zeros(shape, np.float32)
    for r in range(shape[0]):
        cols = rng.choice(shape[1], size=min(nnz, shape[1]), replace=False)
        out[r, cols] = rng.integers(lo, hi + 1, size=len(cols))
    return out


def policy_params(rng, S, H, I, nnz=12, w2=(-1, 1), b2=(-3, 3)):
    """DiscreteActor weights of small integers (float32): sparse W1 rows of entries in [-2, 2], b1 in [0, 2], low-
    entropy W2 (entries in w2) and b2 in b2: many natural ties"""
    return {"w1": _sparse_ints(rng, (H, S), nnz, -2, 2), "b1": small_ints(rng, H, 0, 2),
            "w2": small_ints(rng, (I, H), *w2), "b2": small_ints(rng, I, *b2)}


def policy_state(rng, N, S):
    return small_ints(rng, (N, S), -1, 1)


def policy_logits(p, state):
    """float64 [N, I]: the exact logits (asserting both conditions for both layers)"""
    h = np.maximum(_layer(state, p["w1"], p["b1"], "policy layer 1"), 0.0)
    return _layer(h, p["w2"], p["b2"], "policy layer 2")


def critic_params(rng, S, A, H, nnz=8):
    """Critic weights of small integers (float32): sparse W1 and W2 rows, w3 and the biases in [-2, 2]"""
    return {"w1": _sparse_ints(rng, (H, S + A), nnz, -2, 2), "b1": small_ints(rng, H, -1, 2),
            "w2": _sparse_ints(rng, (H, H), nnz, -1, 1), "b2": small_ints(rng, H, 0, 2),
            "w3": small_ints(rng, (1, H), -2, 2), "b3": small_ints(rng, 1, -2, 2)}


def critic_q(p, state, table):
    """float64 [N, n_items]: the exact Q of every (row, item) pair in the split form the kernels use, u_r + v_j"""
    state, table = np.asarray(state, np.float64), np.asarray(table, np.float64)
    S = state.shape[1]
    u = _layer(state, p["w1"][:, :S], p["b1"], "critic row term")
    v = _layer(table, p["w1"][:, S:], np.zeros(p["w1"].shape[0]), "critic item term")
    # u_r + v_j: exact when |u| + |v| bounds stay below 2^24 (they are sums of the same terms as layer 1)
    both = (np.abs(state) @ np.abs(p["w1"][:, :S]).T + np.abs(p["b1"])).max() + \
        (np.abs(table) @ np.abs(p["w1"][:, S:]).T).max()
    assert both < SUM, "critic layer 1 can reach 2^24"
    out = np.empty((state.shape[0], table.shape[0]))
    for r in range(state.shape[0]):
        h1 = np.maximum(u[r][None, :] + v, 0.0)
        h2 = np.maximum(_layer(h1, p["w2"], p["b2"], "critic layer 2"), 0.0)
        out[r] = _layer(h2, p["w3"], p["b3"], "critic score")[:, 0]
    return out


# ----------------------------------------------------------------------------- the orders
def keys32(z):
    """fp32 keys fminf(-z, FLT_MAX) of float64 values (exact integers or non-finite): NaN and -inf last"""
    return finite_key(-torch.as_tensor(np.asarray(z)).to(torch.float32))


def eligible(n_rows, n_items, exclude=None, columns=None):
    """bool [n_rows, n_items]: exclude / columns per row id lists (negative entries padding), None: none / all"""
    ok = np.ones((n_rows, n_items), bool) if columns is None else np.zeros((n_rows, n_items), bool)
    for r in range(n_rows):
        if columns is not None:
            c = np.asarray(columns[r], np.int64)
            ok[r, c[c >= 0]] = True
        if exclude is not None:
            e = np.asarray(exclude[r], np.int64)
            ok[r, e[e >= 0]] = False
    return ok


def topk(z, k, exclude=None, columns=None):
    """int64 [N, k]: the stable argsort of keys32(z) over each row's eligible items, -1 past the last one"""
    key = keys32(z).numpy().astype(np.float64)
    ok = eligible(z.shape[0], z.shape[1], exclude, columns)
    key = np.where(ok, key, np.inf)                     # an ineligible item sorts after every eligible key (<= FLT_MAX)
    order = np.argsort(key, axis=1, kind="stable")[:, :k]
    keep = np.take_along_axis(ok, order, 1)
    return np.where(keep, order, -1)


def rank(z, target, exclude=None, columns=None):
    """int64 [N]: the eligible j != t with (key_j, j) < (key_t, t); the target is never excluded, and a target outside
    its row's columns gets the row's eligible count"""
    key = keys32(z).numpy()
    target = np.asarray(target, np.int64)
    ok = eligible(z.shape[0], z.shape[1], exclude, columns)
    ids = np.arange(z.shape[1])
    out = np.empty(len(target), np.int64)
    for r, t in enumerate(target):
        inside = columns is None or t in set(np.asarray(columns[r]).tolist())
        if not inside:
            out[r] = ok[r].sum()
            continue
        kt = key[r, t]
        beats = (key[r] < kt) | ((key[r] == kt) & (ids < t))
        out[r] = (beats & ok[r] & (ids != t)).sum()
    return out


# ----------------------------------------------------------------------------- probabilities
def softmax64(z):
    """float64 softmax over each row's finite logits (a -inf logit has probability 0); NaN anywhere: NaN"""
    z = np.asarray(z, np.float64)
    with np.errstate(invalid="ignore", over="ignore"):
        M = np.max(np.where(np.isnan(z), -np.inf, z), 1, keepdims=True)
        e = np.exp(z - M)
        return e / e.sum(1, keepdims=True)


def exact_pi_rows(z):
    """(bool [N], fp32 [N, I]): the rows whose finite logits are all either their max M or at most M - 128 (and hold
    no NaN), and their exact pi: fp32(1 / c) on the c items at M, 0 elsewhere"""
    z = np.asarray(z, np.float64)
    with np.errstate(invalid="ignore"):
        M = np.max(np.where(np.isnan(z), -np.inf, z), 1, keepdims=True)
        top = z == M
        ok = (top | (z <= M - 128) | (z == -np.inf)).all(1) & ~np.isnan(z).any(1) & np.isfinite(M[:, 0])
    c = top.sum(1, keepdims=True).astype(np.float32)
    pi = np.where(top, np.float32(1.0) / np.maximum(c, 1), np.float32(0.0)).astype(np.float32)
    return ok, pi


def pi_bar(z, n_chunks):
    """Relative bound on |fp32 pi - float64 pi| of a row of exact logits z visited in n_chunks chunks:

    - every __expf term exp(d), d = z - m <= 0: (2 + 1.173 |d|) ulp (CUDA's documented bound), and its thread's
      rescale by __expf(m - M) as much again; D = the row's largest finite M - z bounds |d|;
    - the positive sums: a thread adds ceil(I / 256) terms, the block sum 8 levels, the chunk merge one add, a
      relative 2^-24 each;
    - the chunk merge's two expf and two multiplies per chunk, the final expf and the division: 2^-23 each."""
    z = np.asarray(z, np.float64)
    fin = np.where(np.isfinite(z), z, np.nan)
    D = np.nanmax(np.nanmax(fin, 1) - np.nanmin(fin, 1))
    I = z.shape[1]
    terms = 2 * (2 + 1.173 * D) * 2.0 ** -23
    sums = (math.ceil(I / TOPK_THREADS) + 8 + n_chunks) * 2.0 ** -24
    rest = (4 * n_chunks + 3) * 2.0 ** -23
    return 2 * (terms + sums + rest)


# ----------------------------------------------------------------------------- where the selectors cut a row
def topk_splits(n_rows, n_items, cap=SPLIT_CAP):
    """topk.cuh topk_splits: column ranges per row of an [n_rows, n_items] block"""
    s = -(-2 * NUM_SMS // n_rows)
    s = min(s, -(-n_items // (4 * TOPK_THREADS)), cap)
    return max(1, s)


def split_edges(n_rows, n_items, chunk=None, cap=SPLIT_CAP):
    """sorted first ids of every chunk and every column range of a chunked select over n_items items"""
    chunk = n_items if chunk is None or chunk >= n_items else chunk
    edges = set()
    for c0 in range(0, n_items, chunk):
        w = min(chunk, n_items - c0)
        s = topk_splits(n_rows, w, cap)
        per = -(-w // s)
        edges.update(c0 + sp * per for sp in range(s) if sp * per < w)
    return sorted(edges)


def around(edges, n_items):
    """the ids on both sides of every edge"""
    return sorted({e + d for e in edges for d in (-1, 0) if 0 <= e + d < n_items})


def shard_edges(n_items, world):
    per = -(-n_items // world)
    return [min(q * per, n_items) for q in range(world)]
