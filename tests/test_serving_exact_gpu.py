"""Policy and critic serving on integer nets (tests/_exact_serving.py): every logit and every Q is exact on both GEMM
back ends, so ``DiscreteActor.topk`` / ``sample_topk`` / ``rank`` / ``log_prob`` and ``Critic.topk`` / ``rank`` are
compared by equality only -- ids, ranks, the bits of Q and of the probabilities of rows built to be exact -- with ties
planted on both sides of every chunk, column-range and shard edge, at the k-th boundary and deep in the list, and with
-inf and NaN logits."""
from __future__ import annotations

import hashlib
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import recnn_b200
from recnn_b200 import _lib
from recnn_b200.data import ItemSets
from recnn_b200.nn.arena import param_arena
from tests import _exact_serving as X
from tests import _policy_sample_oracle as PS
from tests._discrete import make_policy
from tests._ranks import chunked, returned, run_ranks, shard

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
L = _lib.lib()
KS = (1, 16, 17, 64)
# below fp32's smallest normal a probability (and an __expf term, flushed to 0) keeps no relative precision
TINY = 2.0 ** -120


def _t(x):
    return torch.from_numpy(np.ascontiguousarray(x)).to(DEV)


def _ws(nbytes):
    assert nbytes > 0
    return torch.empty(nbytes, dtype=torch.uint8, device=DEV)


def call_topk(m, st, k, chunk=None, exclude=None, sample_seed=None, row0=0):
    """(values, ids) of one recnn_discrete_topk (or, with sample_seed, recnn_discrete_sample_topk) call"""
    d, n = m.dims, st.shape[0]
    chunk = d.num_items if chunk is None or chunk >= d.num_items else chunk
    nbytes = L.recnn_discrete_topk_workspace_bytes(d, n, k, chunk)
    ws = _ws(nbytes)
    values = torch.empty(n, k, device=DEV)
    ids = torch.empty(n, k, dtype=torch.int64, device=DEV)
    flag = torch.full((1,), 7, dtype=torch.int32, device=DEV)
    ex = None if exclude is None else _t(np.asarray(exclude, np.int64))
    n_ex = 0 if ex is None else ex.shape[1]
    if sample_seed is None:
        _lib.check(L.recnn_discrete_topk(d, param_arena(m).data_ptr(), st.data_ptr(), n, k, _lib.ptr(ex), n_ex, chunk,
                                         values.data_ptr(), ids.data_ptr(), flag.data_ptr(), ws.data_ptr(), nbytes,
                                         _lib.stream_ptr()))
    else:
        _lib.check(L.recnn_discrete_sample_topk(d, param_arena(m).data_ptr(), st.data_ptr(), n, k, _lib.ptr(ex),
                                                n_ex, sample_seed, row0, chunk, values.data_ptr(), ids.data_ptr(),
                                                flag.data_ptr(), ws.data_ptr(), nbytes, _lib.stream_ptr()))
    torch.cuda.synchronize()
    assert int(flag) == 0
    return values, ids


def call_rank(m, st, target, chunk=None):
    """(rank, log_prob) of one recnn_discrete_rank call"""
    d, n = m.dims, st.shape[0]
    chunk = d.num_items if chunk is None or chunk >= d.num_items else chunk
    nbytes = L.recnn_discrete_rank_workspace_bytes(d, n, chunk)
    ws = _ws(nbytes)
    rank = torch.empty(n, dtype=torch.int64, device=DEV)
    logp = torch.empty(n, device=DEV)
    flag = torch.full((1,), 7, dtype=torch.int32, device=DEV)
    tgt = _t(np.asarray(target, np.int64))
    _lib.check(L.recnn_discrete_rank(d, param_arena(m).data_ptr(), st.data_ptr(), tgt.data_ptr(), n, chunk,
                                     rank.data_ptr(), logp.data_ptr(), flag.data_ptr(), ws.data_ptr(), nbytes,
                                     _lib.stream_ptr()))
    torch.cuda.synchronize()
    assert int(flag) == 0
    return rank, logp


class Digest:
    """sha256 of every output a sweep produced, so that two processes (two GEMM back ends) compare bit for bit"""

    def __init__(self):
        self.h = hashlib.sha256()

    def add(self, *ts):
        for t in ts:
            self.h.update(t.detach().contiguous().cpu().numpy().tobytes())

    def hex(self):
        return self.h.hexdigest()


def check_values(values, ids, z, n_chunks, what=""):
    """values of ids: 0 at padding; on exact-pi rows the bits of fp32(1 / c) or 0, elsewhere float64 softmax within
    pi_bar (relative), and exactly 0 for a -inf logit"""
    v, i = values.cpu().numpy(), ids.cpu().numpy()
    assert (v[i < 0] == 0).all(), what
    exact, pi_exact = X.exact_pi_rows(z)
    p64 = X.softmax64(z)
    got_p = np.take_along_axis(p64, np.maximum(i, 0), 1)
    bar = X.pi_bar(z, n_chunks)
    live = i >= 0
    zi = np.take_along_axis(z, np.maximum(i, 0), 1)
    assert (v[live & (zi == -np.inf)] == 0).all(), what
    if exact.any():
        want = np.take_along_axis(pi_exact, np.maximum(i, 0), 1)
        e = exact[:, None] & live
        assert np.array_equal(v[e].view(np.int32), want[e].view(np.int32)), what
    finite = live & np.isfinite(zi)
    assert np.isfinite(v[finite]).all(), (what, v[finite][~np.isfinite(v[finite])][:5])
    err = np.abs(v[finite] - got_p[finite])
    assert (err <= bar * got_p[finite] + TINY).all(), (what, float((err / np.maximum(got_p[finite], 1e-300)).max()), bar)


def _plant(p, ids, anchor, bias=None):
    """copy W2[anchor] and its bias onto ids (exact ties), the bias optionally replaced"""
    p["w2"][ids] = p["w2"][anchor]
    p["b2"][ids] = p["b2"][anchor] if bias is None else bias


def policy_case(S, H, I, N, seed, chunks, lift=True):
    """(p, state, z, top group): low-entropy integer weights; one tie group straddling every chunk and column-range
    edge of `chunks`, lifted above every other logit when it is shorter than 48 (lift), another at the anchor's natural
    place, copies deep inside"""
    rng = np.random.default_rng(seed)
    p = X.policy_params(rng, S, H, I)
    state = X.policy_state(rng, N, S)
    edges = set()
    for c in chunks:
        edges.update(X.split_edges(N, I, c))
    around = X.around(sorted(edges - {0}), I)
    top = [e for e in around if e % 2 == 0] + [0, I - 1]
    natural = [e for e in around if e % 2 == 1] + [I // 3, I // 3 + 1, 2 * I // 3]
    top, natural = sorted(set(top)), sorted(set(natural) - set(top))
    _plant(p, natural, natural[0])
    _plant(p, top, top[0])
    if lift and len(top) < 48:
        z = X.policy_logits(p, state)
        rest = np.delete(z, top, 1).max()
        p["b2"][top] += float(np.ceil(rest - z[:, top[0]].min())) + 1
    return p, state, X.policy_logits(p, state), top


def item_sets(rng, N, I, tied, n_ids):
    """per-row exclusion lists holding tied ids from both sides of edges, and random ids; some rows empty"""
    lists = []
    for r in range(N):
        if r % 5 == 4:
            lists.append([])
            continue
        t = [x for j, x in enumerate(tied) if (j + r) % 3 == 0]
        lists.append(sorted(set(t) | set(rng.choice(I, n_ids, replace=False).tolist())))
    return lists


def dense(lists, E):
    out = np.full((len(lists), E), -1, np.int64)
    for r, l in enumerate(lists):
        l = l[:E]
        out[r, :len(l)] = l
    return out


# (S, H, items, rows, chunkings): S % 4 == 0 and != 0; 1, 7 and 31 column ranges; 70,000 rows (gridDim.y loops)
POLICY = [(52, 32, 1003, 40, (None, 128, 256)), (37, 48, 7000, 40, (None, 256)), (36, 32, 40000, 8, (None, 128)),
          (20, 16, 300, 70000, (None,))]


def run_policy_sweep(digest):
    for S, H, I, N, chunks in POLICY:
        p, state, z, top = policy_case(S, H, I, N, S + I, chunks)
        m = make_policy(p, S, H, I)
        st = _t(state)
        rng = np.random.default_rng(I)
        lists = item_sets(rng, N, I, top, 40)
        ks = KS if N < 10000 else (17,)
        for chunk in chunks:
            nc = -(-I // (chunk or I))
            for k in ks:
                v, i = call_topk(m, st, k, chunk)
                assert np.array_equal(i.cpu().numpy(), X.topk(z, k)), (S, I, chunk, k)
                check_values(v, i, z, nc, (S, I, chunk, k))
                digest.add(v, i)
                if N < 10000 and k in (17, 64):
                    ex = dense(lists, 256)
                    v, i = call_topk(m, st, k, chunk, ex)
                    assert np.array_equal(i.cpu().numpy(), X.topk(z, k, ex)), (S, I, chunk, k, "dense")
                    check_values(v, i, z, nc, (S, I, chunk, k, "dense"))
                    digest.add(v, i)
        if N < 10000:
            sets = ItemSets.from_lists(lists, device=DEV)
            for k in (17, 64):
                v, i = m.topk(st, k, exclude=sets)
                assert np.array_equal(i.cpu().numpy(), X.topk(z, k, lists)), (S, I, k, "sets")
                digest.add(v, i)
        print("policy topk S %d I %d N %d: ok" % (S, I, N))


_DIGESTS = {}          # the tensor-core run's digest of each sweep, for the CUDA-core comparison


def test_policy_topk_ids_and_values():
    d = Digest()
    run_policy_sweep(d)
    _DIGESTS["policy"] = d.hex()


def test_policy_topk_k_at_and_above_the_eligible_count():
    """an ItemSets exclusion leaving e eligible items, tied ones among them: k = e and k > e end in -1 / 0 pads"""
    S, H, I, N = 37, 32, 1003, 24
    p, state, z, top = policy_case(S, H, I, N, 3, (None, 128))
    m = make_policy(p, S, H, I)
    st = _t(state)
    keep = sorted(set(top[::2]) | set(range(500, 520)))
    lists = [sorted(set(range(I)) - set(keep))] * N
    sets = ItemSets.from_lists(lists, device=DEV)
    for k in (len(keep), 64):
        for chunk in (None, 128):
            with chunked(N, chunk):
                v, i = m.topk(st, k, exclude=sets)
            want = X.topk(z, k, lists)
            assert np.array_equal(i.cpu().numpy(), want), (k, chunk)
            assert (want[:, len(keep):] == -1).all()
            check_values(v, i, z, -(-I // (chunk or I)), (k, chunk))


def test_policy_exact_probabilities():
    """rows whose logits are M or <= M - 128: pi is fp32(1 / c) and 0 bit for bit, at every chunking; with one item at
    M, rank's and log_prob's log pi are za - M exactly"""
    S, H, I, N = 52, 32, 1003, 40
    for single in (False, True):
        p, state, z, top = policy_case(S, H, I, N, 9, (None, 128, 256))
        grp = top[:1] if single else top
        p["b2"][grp] += 200
        z = X.policy_logits(p, state)
        exact, pi = X.exact_pi_rows(z)
        assert exact.all()
        m = make_policy(p, S, H, I)
        st = _t(state)
        for chunk in (None, 128, 256):
            v, i = call_topk(m, st, 64, chunk)
            want = np.take_along_axis(pi, i.cpu().numpy(), 1)
            assert np.array_equal(v.cpu().numpy().view(np.int32), want.view(np.int32)), (single, chunk)
        probs = m(st).cpu().numpy()
        assert np.array_equal(probs.view(np.int32), pi.view(np.int32))
        tgt = np.array([grp[0] if r % 2 else (r * 37) % I for r in range(N)])
        for chunk in (None, 128):
            rank, logp = call_rank(m, st, tgt, chunk)
            assert np.array_equal(rank.cpu().numpy(), X.rank(z, tgt))
            lp = m.log_prob(st, _t(tgt))
            assert np.array_equal(logp.cpu().numpy().view(np.int32), lp.cpu().numpy().view(np.int32))
            if single:
                za = np.take_along_axis(z, tgt[:, None], 1)[:, 0]
                want = (za - z.max(1)).astype(np.float32)
                assert np.array_equal(logp.cpu().numpy().view(np.int32), want.view(np.int32)), chunk


def targets(z, top64, seed):
    """per row: a top-k id, a tied id inside a tie group, an id far past the list, the anchor of a tie group"""
    rng = np.random.default_rng(seed)
    N, I = z.shape
    out = np.empty(N, np.int64)
    key = X.keys32(z).numpy()
    for r in range(N):
        c = r % 4
        if c == 0:
            out[r] = top64[r, rng.integers(0, 64)]
        elif c == 1:                                      # the largest id of a tie group of the row
            vals, counts = np.unique(key[r], return_counts=True)
            g = vals[counts > 1][rng.integers(0, (counts > 1).sum())]
            out[r] = np.nonzero(key[r] == g)[0].max()
        elif c == 2:
            out[r] = np.argsort(key[r], kind="stable")[rng.integers(I // 2, I)]
        else:
            out[r] = rng.integers(0, I)
    return out


def test_policy_rank_and_log_prob():
    for S, H, I, N, chunks in POLICY[:3]:
        p, state, z, top = policy_case(S, H, I, N, 2 * S + I, chunks, lift=False)
        m = make_policy(p, S, H, I)
        st = _t(state)
        top64 = X.topk(z, 64)
        tgt = targets(z, top64, S)
        want = X.rank(z, tgt)
        p64 = X.softmax64(z)
        for chunk in chunks:
            with chunked(N, chunk):
                rank, logp = m.rank(st, _t(tgt))
                lp = m.log_prob(st, _t(tgt))
                _, ids = m.topk(st, 64)
            assert np.array_equal(rank.cpu().numpy(), want), (I, chunk)
            assert np.array_equal(logp.cpu().numpy().view(np.int32), lp.cpu().numpy().view(np.int32)), (I, chunk)
            ids = ids.cpu().numpy()
            for r in range(N):
                hit = np.nonzero(ids[r] == tgt[r])[0]
                assert (hit[0] if hit.size else 64) == min(want[r], 64), (I, chunk, r)
            lt = np.log(p64[np.arange(N), tgt])
            assert (np.abs(logp.cpu().numpy() - lt) <= 2 * X.pi_bar(z, -(-I // (chunk or I)))).all(), (I, chunk)
        # the target inside its own exclusion set is still ranked, never excluded; the tied ids of the set do not count
        lists = item_sets(np.random.default_rng(1), N, I, top, 30)
        lists = [sorted(set(l) | {int(tgt[r])}) for r, l in enumerate(lists)]
        rank, _ = m.rank(st, _t(tgt), exclude=ItemSets.from_lists(lists, device=DEV))
        assert np.array_equal(rank.cpu().numpy(), X.rank(z, tgt, [[x for x in l if x != tgt[r]]
                                                                   for r, l in enumerate(lists)])), I


# ----------------------------------------------------------------------------- sampled slates
def test_sample_ids_are_invariant_and_values_are_topk_bits():
    S, H, I, N, seed = 52, 32, 1003, 40, 12345
    p, state, z, top = policy_case(S, H, I, N, 77, (None, 128, 256), lift=False)
    m = make_policy(p, S, H, I)
    st = _t(state)
    v0, i0 = call_topk(m, st, 64, None, sample_seed=seed)
    probs = m(st)
    assert torch.equal(v0, probs.gather(1, i0))
    for chunk in (128, 256):
        v, i = call_topk(m, st, 64, chunk, sample_seed=seed)
        assert torch.equal(i, i0), chunk
        tv, ti = call_topk(m, st, 64, chunk)
        for r in range(N):
            both = np.intersect1d(i[r].cpu().numpy(), ti[r].cpu().numpy())
            a = v[r][torch.isin(i[r], _t(both))].cpu().numpy()
            b = tv[r][torch.isin(ti[r], _t(both))].cpu().numpy()
            ia = i[r][torch.isin(i[r], _t(both))].cpu().numpy()
            ib = ti[r][torch.isin(ti[r], _t(both))].cpu().numpy()
            assert np.array_equal(a[np.argsort(ia)].view(np.int32), b[np.argsort(ib)].view(np.int32)), (chunk, r)
    half = N // 2                                                   # batching and row offsets
    _, ia = call_topk(m, st[:half], 64, 128, sample_seed=seed, row0=0)
    _, ib = call_topk(m, st[half:], 64, 256, sample_seed=seed, row0=half)
    assert torch.equal(torch.cat([ia, ib]), i0)
    ex = dense(item_sets(np.random.default_rng(2), N, I, top, 50), 128)
    _, ie = call_topk(m, st, 17, 128, ex, sample_seed=seed)
    _, ie2 = call_topk(m, st, 17, None, ex, sample_seed=seed)
    assert torch.equal(ie, ie2)
    assert not any(np.isin(ie[r].cpu().numpy(), ex[r][ex[r] >= 0]).any() for r in range(N))


def test_sample_against_the_float64_draw():
    """logits within a few units, so the noise decides the order: the settled slots (by a bar that covers only G's
    fp32 rounding, the logits being exact) must be the float64 draw's, and nearly every slot is settled"""
    S, H, I, N, k, seed = 36, 32, 2000, 64, 16, 99
    rng = np.random.default_rng(5)
    p = X.policy_params(rng, S, H, I, nnz=2, w2=(0, 0), b2=(-4, 0))
    p["w2"][:, :2] = X.small_ints(rng, (I, 2), -1, 1)             # |z| <= 16: two hidden units reach the logits
    state = X.policy_state(rng, N, S)
    z = X.policy_logits(p, state)
    m = make_policy(p, S, H, I)
    _, ids = call_topk(m, _t(state), k, 256, sample_seed=seed)
    _, want_i, top_g = PS.sample_topk(z, k + 1, seed)
    # fp32 G = -logf(-logf(u)): two logs of 1 ulp each and the sum z + G's rounding, with |G| <= 16.75
    bar = 4 * 2.0 ** -23 * (1 + PS.G_MAX + np.abs(z).max())
    slot, _ = PS.determined(top_g, k, bar)
    got = ids.cpu().numpy()
    assert slot.mean() >= 0.99, slot.mean()
    assert (got[slot] == want_i[:, :k][slot]).all()


# ----------------------------------------------------------------------------- vocabulary-parallel
def sharded(full, world, fn, chunk=None, rows=None):
    def rank(r):
        pol = shard({"policy_net": full})[0]["policy_net"]
        return fn(pol)
    with chunked(rows, chunk):
        return returned(run_ranks(world, rank))


@pytest.mark.parametrize("world", [1, 2, 3, 8])
def test_virtual_ranks(world):
    for S, H, I, N in [(52, 32, 1003, 24), (37, 32, 200, 17)]:      # 200 items over 8 ranks: 25 per block < k
        rng = np.random.default_rng(I + world)
        p = X.policy_params(rng, S, H, I)
        state = X.policy_state(rng, N, S)
        edges = X.around([e for e in X.shard_edges(I, world) if e] + X.split_edges(N, I, 128)[1:], I)
        _plant(p, edges[::2], edges[0])
        _plant(p, edges[1::2], edges[1])
        z = X.policy_logits(p, state)
        full = make_policy(p, S, H, I)
        st = _t(state)
        tgt = targets(z, X.topk(z, 64), world)
        for chunk in (None, 128):
            for k in (17, 64):
                res = sharded(full, world, lambda pol: pol.topk(st, k) + pol.sample_topk(st, k, seed=7), chunk, N)
                for x in res[1:]:
                    assert all(torch.equal(a, b) for a, b in zip(x, res[0]))
                v, i, sv, si = res[0]
                assert np.array_equal(i.cpu().numpy(), X.topk(z, k)), (world, I, chunk, k)
                with chunked(N, chunk):
                    one_v, one_i = full.topk(st, k)
                    one_sv, one_si = full.sample_topk(st, k, seed=7)
                assert torch.equal(i, one_i) and torch.equal(si, one_si), (world, I, chunk, k)
                check_values(v, i, z, world * 8, (world, I, chunk, k))
                if world == 1:
                    assert torch.equal(v, one_v) and torch.equal(sv, one_sv)
            ranks = sharded(full, world, lambda pol: pol.rank(st, _t(tgt)), chunk, N)
            assert np.array_equal(ranks[0][0].cpu().numpy(), X.rank(z, tgt)), (world, I, chunk)


# ----------------------------------------------------------------------------- non-finite logits
def _masked(p, state, ids, value):
    q = {k: v.copy() for k, v in p.items()}
    q["b2"][ids] = value
    return q, X.policy_logits(q, state)


def nonfinite_cases(I, chunk, world, boundary):
    """{name: ids whose bias is set non-finite}"""
    per = -(-I // world)
    return {"id 0": [0], "ids 0..255": list(range(256)), "a whole chunk": list(range(chunk, 2 * chunk)),
            "the first two chunks": list(range(2 * chunk)), "a shard block": list(range(per, 2 * per)),
            "the k-th boundary": boundary}


def test_minus_inf_logits():
    """b2 = -inf masks items: they rank after every finite logit (ties by id) and before any pad, their value is 0,
    and forward, every other value, rank and log_prob are float64's softmax over the finite logits, finite"""
    S, H, I, N, k, chunk, world = 36, 32, 1003, 24, 17, 128, 3
    p, state, z, top = policy_case(S, H, I, N, 21, (None, chunk), lift=False)
    boundary = X.topk(z, k + 2)[0, k - 2:k + 2].tolist()
    cases = nonfinite_cases(I, chunk, world, boundary)
    failures = []
    for name, ids in cases.items():
        q, zq = _masked(p, state, ids, -np.inf)
        m = make_policy(q, S, H, I)
        st = _t(state)
        tgt = np.array([ids[r % len(ids)] if r % 3 == 0 else (r * 41) % I for r in range(N)])
        p64 = X.softmax64(zq)
        with np.errstate(divide="ignore"):
            lt = np.log(p64[np.arange(N), tgt])
        for c in (None, chunk):
            nc = -(-I // (c or I))
            with chunked(N, c):
                v, i = m.topk(st, 64)
                sv, si = m.sample_topk(st, 64, seed=3)
                rank, logp = m.rank(st, _t(tgt))
                lp = m.log_prob(st, _t(tgt))
            got = {"topk values": v.cpu().numpy(), "sample values": sv.cpu().numpy(), "log_prob": lp.cpu().numpy()}
            fin = np.isfinite(lt)
            bad = [w for w, a in got.items() if np.isnan(a).any()]
            if bad:
                failures.append((name, c, bad, got["topk values"][0, :4].tolist(), got["log_prob"][:4].tolist()))
                continue
            assert np.array_equal(i.cpu().numpy(), X.topk(zq, 64)), (name, c)
            check_values(v, i, zq, nc, (name, c))
            check_values(sv, si, zq, nc, (name, c, "sample"))
            assert np.array_equal(rank.cpu().numpy(), X.rank(zq, tgt)), (name, c)
            assert np.array_equal(logp.cpu().numpy().view(np.int32), lp.cpu().numpy().view(np.int32)), (name, c)
            assert (got["log_prob"][~fin] == -np.inf).all(), (name, c)
            assert (np.abs(got["log_prob"][fin] - lt[fin]) <= 2 * X.pi_bar(zq, nc)).all(), (name, c)
        probs = m(st).cpu().numpy()
        if np.isnan(probs).any():
            failures.append((name, "forward", probs[0, :4].tolist()))
            continue
        assert (np.abs(probs - p64) <= X.pi_bar(zq, 1) * p64 + TINY).all(), (name, "forward")
        # the same masks on W virtual ranks: the -inf items come before the pads of an exclusion leaving < k
        keep = sorted(set(ids[:40]) | set(range(700, 710)))
        lists = [sorted(set(range(I)) - set(keep))] * N
        sets = ItemSets.from_lists(lists, device=DEV)
        res = sharded(m, world, lambda pol: pol.topk(st, 64, exclude=sets), chunk, N)
        if np.isnan(res[0][0].cpu().numpy()).any():
            failures.append((name, "sharded", res[0][0][0, :4].tolist()))
            continue
        want = X.topk(zq, 64, lists)
        assert np.array_equal(res[0][1].cpu().numpy(), want), (name, "sharded")
        assert (want[:, :len(keep)] >= 0).all() and (want[:, len(keep):] == -1).all()
        check_values(res[0][0], res[0][1], zq, 8, (name, "sharded"))
    assert not failures, failures


def test_nan_logits():
    """b2 = NaN: the items rank as -inf ones do (after every finite logit, ties by id, before pads) and every value
    is NaN, as torch.softmax gives"""
    S, H, I, N = 36, 32, 1003, 24
    p, state, z, top = policy_case(S, H, I, N, 23, (None, 128), lift=False)
    nan_ids = [5, 300, 301, 640, 1002]
    q, zq = _masked(p, state, nan_ids, np.nan)
    m = make_policy(q, S, H, I)
    st = _t(state)
    lists = [sorted(set(range(I)) - set(nan_ids) - set(range(100, 120)))] * N
    sets = ItemSets.from_lists(lists, device=DEV)
    for c in (None, 128):
        with chunked(N, c):
            v, i = m.topk(st, 64)
            ve, ie = m.topk(st, 30, exclude=sets)
        assert np.array_equal(i.cpu().numpy(), X.topk(zq, 64)), c
        want = X.topk(zq, 30, lists)
        assert np.array_equal(ie.cpu().numpy(), want), c
        assert (want[:, 20:25] == np.array(nan_ids)).all() and (want[:, 25:] == -1).all()
        assert np.isnan(v.cpu().numpy()).all() and np.isnan(ve.cpu().numpy()[:, :25]).all(), c
    assert torch.isnan(m(st)).all()


# ----------------------------------------------------------------------------- critic
# (S, A, H, items, rows): the canonical critic on the tensor cores, a ragged one on the CUDA cores (H % 4 != 0)
CRITIC = [(1290, 128, 256, 3000, 24), (37, 13, 30, 700, 9)]


def critic_case(S, A, H, I, N, seed):
    rng = np.random.default_rng(seed)
    p = X.critic_params(rng, S, A, H)
    state = X.small_ints(rng, (N, S), -1, 1)
    table = X.small_ints(rng, (I, A), -1, 1)
    edges = set()
    for c in (7, 128, 4096):
        edges.update(range(0, I, c))
    edges.update(X.split_edges(N, I, None))
    around = X.around(sorted(edges - {0}), I)
    for grp in (around[::2], around[1::2]):
        table[grp] = table[grp[0]]
    c = recnn_b200.nn.Critic(S, A, H)
    with torch.no_grad():
        for name, lin in (("1", c.linear1), ("2", c.linear2), ("3", c.linear3)):
            lin.weight.copy_(torch.from_numpy(p["w" + name]))
            lin.bias.copy_(torch.from_numpy(p["b" + name]))
    return c.to(DEV).eval(), state, table, X.critic_q(p, state, table), around


def run_critic_sweep(digest):
    for S, A, H, I, N in CRITIC:
        c, state, table, q, tied = critic_case(S, A, H, I, N, S + I)
        st, tb = _t(state), _t(table)
        rng = np.random.default_rng(I)
        rest = np.setdiff1d(np.arange(I), tied[:19])               # 19 tied ids and 281 others, no repeats
        cands = np.stack([np.concatenate([tied[:19], rng.permutation(rest)[:281]]) for _ in range(N)])
        cands[:, 20::7] = -1
        lists = item_sets(rng, N, I, tied, 20)
        sets = ItemSets.from_lists(lists, device=DEV)
        tgt = np.array([cands[r, 5] if r % 3 else rng.integers(0, I) for r in range(N)])
        for chunk in (7, 128, None):
            for mode, cols in (("all", None), ("cand", cands)):
                ct = None if cols is None else _t(cols)
                for k in (1, 17, 64):
                    v, i = c.topk(st, k, tb, candidates=ct, exclude=sets, chunk=chunk)
                    want = X.topk(q, k, lists, cols)
                    got = i.cpu().numpy()
                    assert np.array_equal(got, want), (S, chunk, mode, k)
                    qv = np.where(want >= 0, np.take_along_axis(q, np.maximum(want, 0), 1), -X.FLT_MAX)
                    assert np.array_equal(v.cpu().numpy().view(np.int32), qv.astype(np.float32).view(np.int32))
                    digest.add(v, i)
                rk = c.rank(st, _t(tgt), tb, candidates=ct, exclude=sets, chunk=chunk)
                ex = [[x for x in l if x != tgt[r]] for r, l in enumerate(lists)]
                assert np.array_equal(rk.cpu().numpy(), X.rank(q, tgt, ex, cols)), (S, chunk, mode)
                digest.add(rk)
        print("critic S %d I %d: ok" % (S, I))


def test_critic_topk_and_rank():
    d = Digest()
    run_critic_sweep(d)
    _DIGESTS["critic"] = d.hex()


# ----------------------------------------------------------------------------- both back ends
def sweep_digests():
    out = []
    for name, run in (("policy", run_policy_sweep), ("critic", run_critic_sweep)):
        d = Digest()
        run(d)
        out.append(d.hex())
    return out


def test_cuda_core_back_end_returns_the_same_bits():
    """the sweeps with every GEMM on the exact-fp32 CUDA-core kernel, in a process of its own (the back end is fixed
    per process): every id, rank and value equal to the tensor-core run's bits"""
    code = ("import sys; sys.path.insert(0, %r); from tests import test_serving_exact_gpu as T; "
            "print('DIGEST', *T.sweep_digests())" % ROOT)
    env = dict(os.environ, RECNN_B200_MATH="simt")
    r = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, cwd=ROOT)
    print(r.stdout[-2000:], r.stderr[-3000:])
    assert r.returncode == 0
    simt = [l for l in r.stdout.splitlines() if l.startswith("DIGEST")][0].split()[1:]
    tc = [_DIGESTS.get("policy"), _DIGESTS.get("critic")]
    if None in tc:                     # run alone: make the tensor-core digests here
        tc = sweep_digests()
    assert simt == tc


# ----------------------------------------------------------------------------- scale
def test_million_items():
    """2^20 items, H = 32, 64 rows: topk and rank against a float64 oracle on the device"""
    S, H, I, N, k = 40, 32, 1 << 20, 64, 64
    rng = np.random.default_rng(8)
    p = X.policy_params(rng, S, H, I)
    edges = X.around(X.split_edges(N, I, None)[1:], I)
    _plant(p, edges, edges[0])
    state = X.policy_state(rng, N, S)
    h = np.maximum(X._layer(state, p["w1"], p["b1"], "layer 1"), 0)
    assert (np.abs(h).sum(1) * 1 + 3 < X.SUM).all() and np.abs(h).max() <= X.OPERAND
    m = make_policy(p, S, H, I)
    st = _t(state)
    v, i = m.topk(st, k)
    with torch.no_grad():
        z = _t(h).double() @ _t(p["w2"]).double().T + _t(p["b2"]).double()
        key = X.finite_key(-z.float())
        order = torch.sort(key, dim=1, stable=True).indices[:, :k]
    assert torch.equal(i, order)
    tgt = order[:, 40].clone()
    tgt[::2] = torch.arange(0, I, I // (N // 2), device=DEV)[:N // 2]
    rank, _ = m.rank(st, tgt)
    kt = key.gather(1, tgt[:, None])
    ids = torch.arange(I, device=DEV)[None, :]
    want = ((key < kt) | ((key == kt) & (ids < tgt[:, None]))).sum(1)
    assert torch.equal(rank, want)
