"""Serving through the DDPG / TD3 critic on the device: ``Critic.topk`` / ``Critic.rank`` against the float64
restatement (tests/_critic_serve_oracle.py) on both GEMM back ends, their exact invariants (chunking, batching, the two
modes, rank == position in topk, ties), exclusion and candidate rules, the critic's state, an end-to-end
actor -> search -> critic run on a DeviceFrameFeed, and memory at a million items."""
from __future__ import annotations

import copy
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import recnn_b200
from recnn_b200.data import DeviceFrameFeed, HistoryCSR, ItemIndex, ItemSets
from recnn_b200.nn.arena import param_arena
from recnn_b200.utils.metrics import ranking_metrics
from tests import _critic_serve_oracle as O
from tests.test_recommend_gpu import make_sets, padded

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
# (S, A, H, items, rows): the canonical ML-20M critic; a ragged one (S % 4 = 1, A odd, H % 4 = 2: the CUDA-core path);
# a small hidden layer on the tensor cores
SHAPES = [(1290, 128, 256, 3000, 24), (37, 13, 30, 700, 9), (20, 8, 16, 500, 11)]
BAR = 5e-5          # |fp32 Q - float64 Q| at these scales (|Q| ~ 1)
FLT_MAX = O.FLT_MAX


def make_case(S, A, H, I, N, seed):
    torch.manual_seed(seed)
    c = recnn_b200.nn.Critic(S, A, H)
    with torch.no_grad():
        c.linear3.weight.uniform_(-0.3, 0.3)
        c.linear3.bias.uniform_(-0.3, 0.3)
    c = c.to(DEV).eval()
    g = torch.Generator().manual_seed(seed + 1)
    state = torch.randn(N, S, generator=g)
    table = torch.randn(I, A, generator=g)
    return c, O.params64(c), state.to(DEV), table.to(DEV), state.double().numpy(), table.double().numpy()


def rand_cands(n, items, m, seed, pad=0.15):
    rng = np.random.default_rng(seed)
    out = np.stack([rng.permutation(items)[:m] for _ in range(n)]).astype(np.int64)
    if m > 1:
        out[rng.random(out.shape) < pad] = -1
    return out


def check_against_float64(vals, ids, q64_of, cols, k, exclude=None, what=""):
    """Q of every returned id within BAR of float64; the returned set is float64's top k on every row whose k-th /
    (k+1)-th gap exceeds 2 BAR; the list is sorted by (Q desc, id asc) in fp32."""
    vals, ids = vals.cpu().numpy(), ids.cpu().numpy()
    sure = 0
    for r in range(ids.shape[0]):
        el = O.order(q64_of[r], cols[r], None if exclude is None else exclude[r])
        got = ids[r][ids[r] >= 0]
        assert got.size == min(k, len(el)), (what, r)
        assert (ids[r][got.size:] == -1).all() and (vals[r][got.size:] == -FLT_MAX).all(), (what, r)
        q_of = {i: q for q, i in el}
        for j, i in enumerate(got):
            assert abs(vals[r, j] - q_of[int(i)]) <= BAR, (what, r, j, vals[r, j], q_of[int(i)])
            if j:
                assert vals[r, j - 1] > vals[r, j] or (vals[r, j - 1] == vals[r, j] and got[j - 1] < i), (what, r, j)
        m = got.size
        if m == len(el) or el[m - 1][0] - el[m][0] > 2 * BAR:
            assert set(got.tolist()) == {i for _, i in el[:m]}, (what, r)
            sure += 1
    assert sure >= ids.shape[0] // 2, (what, sure)


def positions(ids, target):
    ids = ids.cpu().numpy()
    out = np.full(len(target), -1)
    for r, t in enumerate(target):
        hit = np.nonzero(ids[r] == t)[0]
        if hit.size:
            out[r] = hit[0]
    return out


def check_rank_consistency(rank, top64_ids, target, what="", cols=None):
    """rank == the target's position in topk(64) (absent when >= 64); with candidates `cols`, a target missing from
    its row's candidates is absent from the list whatever its rank (the row's eligible count)"""
    rank = rank.cpu().numpy()
    pos = positions(top64_ids, target)
    for r in range(len(target)):
        if cols is not None and target[r] not in set(cols[r].tolist()):
            assert pos[r] == -1, (what, r)
            continue
        assert pos[r] == (rank[r] if rank[r] < 64 else -1), (what, r, rank[r], pos[r])


def targets_for(q64, cols, seed):
    """one target per row: mostly among the row's best columns, some anywhere"""
    rng = np.random.default_rng(seed)
    out = []
    for r in range(cols.shape[0]):
        el = O.order(q64[r], cols[r])
        pick = el[int(rng.integers(0, min(len(el), 40)))][1] if r % 3 else el[int(rng.integers(0, len(el)))][1]
        out.append(pick)
    return np.array(out, np.int64)


# ----------------------------------------------------------------------------- 1. float64, both back ends, all modes
def run_sweep():
    for S, A, H, I, N in SHAPES:
        c, p, st, table, s64, t64 = make_case(S, A, H, I, N, S + I)
        allc = O.all_ids(N, I)
        q_all = O.q_pairs(p, s64, t64, allc, rows_per_step=4)
        lists, rows = make_sets(q_all, 10, S)
        sets = ItemSets.from_lists(lists, device=DEV)
        ex = [[int(x) for x in row if x >= 0] for row in padded(lists, rows)]
        rows_t = torch.from_numpy(rows).to(DEV)
        modes = [("all", None, allc)]
        for m in (1, 10, 64, 300):
            cand = rand_cands(N, I, m, S + m)
            modes.append(("cand%d" % m, torch.from_numpy(cand).to(DEV), cand))
        for name, cand_t, cols in modes:
            q64 = np.take_along_axis(q_all, np.where(cols >= 0, cols, 0), 1)
            q64[cols < 0] = np.nan
            target = targets_for(q64, cols, S)
            if name == "cand300":
                target[::4] = (target[::4] + 1) % I              # some targets missing from their candidates
            tgt = torch.from_numpy(target).to(DEV)
            ref = None
            for chunk in (None, 1, 7):
                v, i = c.topk(st, 10, table, candidates=cand_t, chunk=chunk)
                check_against_float64(v, i, q64, cols, 10, what=(S, name, chunk))
                vx, ix = c.topk(st, 10, table, candidates=cand_t, exclude=sets, exclude_rows=rows_t, chunk=chunk)
                check_against_float64(vx, ix, q64, cols, 10, ex, what=(S, name, chunk, "sets"))
                v64, i64 = c.topk(st, 64, table, candidates=cand_t, chunk=chunk)
                rk = c.rank(st, tgt, table, candidates=cand_t, chunk=chunk)
                check_rank_consistency(rk, i64, target, (S, name, chunk), cols)
                rkx = c.rank(st, tgt, table, candidates=cand_t, exclude=sets, exclude_rows=rows_t, chunk=chunk)
                _, i64x = c.topk(st, 64, table, candidates=cand_t, chunk=chunk,
                                 exclude=ItemSets.from_lists([[x for x in e if x != t] for e, t in zip(ex, target)],
                                                             device=DEV))
                check_rank_consistency(rkx, i64x, target, (S, name, chunk, "sets"), cols)
                want = O.rank(q64, cols, target, ex)
                got = rkx.cpu().numpy()
                sure = 0
                for r in range(N):                               # float64's rank where no Q is within 2 BAR of the target's
                    qs = q64[r][cols[r] >= 0]
                    qt = q64[r][cols[r] == target[r]]
                    gaps = np.sort(np.abs(qs - qt[0]))[1:] if qt.size else np.array([np.inf])
                    if gaps.size == 0 or gaps[0] > 2 * BAR:
                        assert got[r] == want[r], (S, name, chunk, r, got[r], want[r])
                        sure += 1
                assert sure >= N // 2
                out = tuple(t.cpu() for t in (v, i, vx, ix, v64, i64, rk, rkx))
                if ref is None:
                    ref = out
                else:                                            # bit-identical at every chunk width
                    for a, b in zip(ref, out):
                        assert torch.equal(a.view(torch.int32) if a.dtype == torch.float32 else a,
                                           b.view(torch.int32) if b.dtype == torch.float32 else b), (S, name, chunk)
            if name == "all":
                all_ref = ref
                # the two modes agree on the same pairs: candidates = the all-items lists
                cv, ci = c.topk(st, 10, table, candidates=all_ref[5][:, :10].to(DEV))
                assert torch.equal(cv.cpu().view(torch.int32), all_ref[0].view(torch.int32))
                assert torch.equal(ci.cpu(), all_ref[1])
            if name == "cand300":                                # and Q of one pair is the same bits in a list of one
                one = cand_t[:, :1]
                q1, _ = c.topk(st, 1, table, candidates=one)
                ok = (one[:, 0] >= 0).cpu()
                pos = (i64.cpu() == one.cpu()).nonzero()
                for r, j in pos.tolist():
                    assert ok[r] and q1[r, 0].cpu().view(torch.int32) == v64[r, j].cpu().view(torch.int32)
        # every item as candidates, permuted per row: the all-items bits
        perm = torch.stack([torch.randperm(I) for _ in range(N)]).to(DEV)
        pv, pi = c.topk(st, 10, table, candidates=perm)
        assert torch.equal(pv.cpu().view(torch.int32), all_ref[0].view(torch.int32)) and torch.equal(pi.cpu(), all_ref[1])
        print("critic serve S %d A %d H %d: ok" % (S, A, H))


def test_against_float64():
    run_sweep()


def test_against_float64_on_the_cuda_core_back_end():
    code = "import sys; sys.path.insert(0, %r); from tests import test_critic_serve_gpu as T; T.run_sweep()" % ROOT
    env = dict(os.environ, RECNN_B200_MATH="simt")
    r = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, cwd=ROOT)
    print(r.stdout[-3000:], r.stderr[-3000:])
    assert r.returncode == 0


# ----------------------------------------------------------------------------- 2. invariants
@pytest.mark.parametrize("S,A,H,I,N", SHAPES)
def test_repeat_batching_and_ties_across_chunk_edges(S, A, H, I, N):
    c, p, st, table, s64, t64 = make_case(S, A, H, I, N, 3 * S)
    cand = torch.from_numpy(rand_cands(N, I, 64, S)).to(DEV)
    for cd in (None, cand):
        v, i = c.topk(st, 16, table, candidates=cd, chunk=7)
        v2, i2 = c.topk(st, 16, table, candidates=cd, chunk=7)
        assert torch.equal(v.view(torch.int32), v2.view(torch.int32)) and torch.equal(i, i2)
        for r in (0, N // 2, N - 1):
            va, ia = c.topk(st[r:r + 1], 16, table, candidates=None if cd is None else cd[r:r + 1], chunk=5)
            assert torch.equal(va.view(torch.int32), v[r:r + 1].view(torch.int32)) and torch.equal(ia, i[r:r + 1])
    # exact ties: the best item of row 0, duplicated on both sides of chunk edges (chunk 7) -> smallest id first
    _, i = c.topk(st, 1, table)
    best = int(i[0, 0])
    dups = sorted({6, 7, 13, 14, I - 1, best})
    tied = table.clone()
    tied[dups] = table[best]
    for chunk in (None, 7):
        v, i = c.topk(st, 16, tied, chunk=chunk)
        assert i[0, :len(dups)].tolist() == dups
        assert (v[0, :len(dups)].view(torch.int32) == v[0, 0].view(torch.int32)).all()
        for r in range(N):
            row = i[r].tolist()
            at = [j for j, x in enumerate(row) if x in dups]
            assert [row[j] for j in at] == sorted(row[j] for j in at) and at == list(range(at[0], at[0] + len(at))) \
                if at else True
        rk = c.rank(st, torch.full((N,), dups[-1], dtype=torch.int64, device=DEV), tied, chunk=chunk)
        _, i64 = c.topk(st, 64, tied, chunk=chunk)
        check_rank_consistency(rk, i64, [dups[-1]] * N, ("ties", chunk))


# ----------------------------------------------------------------------------- 3. exclusion
def test_exclusion_rules_and_errors():
    S, A, H, I, N = 37, 13, 32, 700, 10
    c, p, st, table, _, _ = make_case(S, A, H, I, N, 11)
    cand = torch.from_numpy(rand_cands(N, I, 100, 5, pad=0.0)).to(DEV)
    for cd in (None, cand):
        _, full = c.topk(st, 64, table, candidates=cd)
        lists = []
        for r in range(N):
            row = full[r].tolist()
            e = [x for x in row[:20] if x % 7 in (0, 6)] + row[:3]     # ids on the chunk-7 edges, and the best three
            lists.append(sorted(set(e)))
        lists[3] = sorted(set(full[3].tolist()) | set(range(I)) if cd is None else set(cd[3].tolist()))  # covers all
        rows = torch.arange(N, device=DEV)
        rows[5] = -1
        sets = ItemSets.from_lists(lists, device=DEV)
        for chunk in (None, 7):
            v, i = c.topk(st, 10, table, candidates=cd, exclude=sets, exclude_rows=rows, chunk=chunk)
            for r in range(N):
                drop = set() if r == 5 else set(lists[r])
                want = [x for x in full[r].tolist() if x not in drop][:10]
                if r == 3:
                    assert (i[r] == -1).all() and (v[r] == -FLT_MAX).all()
                else:
                    assert i[r].tolist() == want, (r, chunk)
    bad = ItemSets.from_lists([[1, 2, 3]] * N, device=DEV)
    bad.ids = bad.ids.flip(0).contiguous()                                   # a descending set
    for call in (lambda **kw: c.topk(st, 5, table, **kw),
                 lambda **kw: c.rank(st, torch.zeros(N, dtype=torch.int64, device=DEV), table, **kw)):
        with pytest.raises(ValueError, match="malformed"):
            call(exclude=bad)
        with pytest.raises(ValueError, match="malformed"):
            call(exclude=ItemSets.from_lists([[1]] * 2, device=DEV), exclude_rows=torch.full((N,), 2, device=DEV))
        with pytest.raises(IndexError):
            call(exclude=ItemSets.from_lists([[1, I]] * N, device=DEV))


# ----------------------------------------------------------------------------- 4. candidates
def test_candidate_rules_and_errors():
    S, A, H, I, N = 20, 8, 16, 500, 6
    c, p, st, table, s64, t64 = make_case(S, A, H, I, N, 12)
    cand = rand_cands(N, I, 40, 3, pad=0.3)
    ct = torch.from_numpy(cand).to(DEV)
    v, i = c.topk(st, 64, table, candidates=ct)
    assert ((i >= 0).sum(1).cpu().numpy() == (cand >= 0).sum(1)).all()       # padding is never returned
    for r in range(N):
        assert set(i[r][i[r] >= 0].tolist()) == set(cand[r][cand[r] >= 0].tolist())
    # an absent target's rank is the eligible count; a target is never excluded
    absent = np.array([next(x for x in range(I) if x not in set(cand[r].tolist())) for r in range(N)])
    rk = c.rank(st, torch.from_numpy(absent).to(DEV), table, candidates=ct)
    assert rk.cpu().numpy().tolist() == (cand >= 0).sum(1).tolist()
    present = np.array([cand[r][cand[r] >= 0][0] for r in range(N)])
    tp = torch.from_numpy(present).to(DEV)
    plain = c.rank(st, tp, table, candidates=ct)
    with_t = c.rank(st, tp, table, candidates=ct, exclude=ItemSets.from_lists([[int(x)] for x in present], device=DEV))
    assert torch.equal(plain, with_t)
    check_rank_consistency(plain, i, present)
    rep = ct.clone()
    rep[2, 5] = rep[2, 30] = 17
    with pytest.raises(ValueError, match="repeated"):
        c.topk(st, 5, table, candidates=rep)
    with pytest.raises(ValueError, match="repeated"):
        c.rank(st, tp, table, candidates=rep)
    for badv in (I, -2):
        b = ct.clone()
        b[1, 3] = badv
        with pytest.raises(IndexError):
            c.topk(st, 5, table, candidates=b)
    with pytest.raises(IndexError):
        c.rank(st, torch.full((N,), I, dtype=torch.int64, device=DEV), table, candidates=ct)
    # a long candidate list (several shared-memory tiles of the repeat check)
    long = torch.stack([torch.randperm(I) for _ in range(N)])[:, :450].repeat(1, 6)[:, :2500]
    long = torch.where(torch.arange(2500) < 450, long, torch.full_like(long, -1)).to(DEV)
    long[0, 2400] = long[0, 0]
    with pytest.raises(ValueError, match="repeated"):
        c.topk(st, 5, table, candidates=long)


# ----------------------------------------------------------------------------- 5. the critic's state
def test_state_untouched_and_train_mode_scores_as_eval():
    S, A, H, I, N = 37, 13, 32, 300, 5
    c, p, st, table, _, _ = make_case(S, A, H, I, N, 13)
    opt = torch.optim.Adam(c.parameters(), lr=1e-3)
    for q in c.parameters():
        q.grad = torch.ones_like(q)
    opt.step()
    arena = param_arena(c).clone()
    grads = [q.grad.clone() for q in c.parameters()]
    ost = copy.deepcopy(opt.state_dict())
    twin = copy.deepcopy(c).eval()
    c.train()
    v, i = c.topk(st, 8, table)
    rk = c.rank(st, i[:, 3].contiguous(), table)
    assert c.training and torch.equal(param_arena(c), arena)
    assert all(torch.equal(q.grad, g) for q, g in zip(c.parameters(), grads))
    now = opt.state_dict()
    for k_, s_ in ost["state"].items():
        for name, t in s_.items():
            assert torch.equal(torch.as_tensor(now["state"][k_][name]), torch.as_tensor(t))
    v2, i2 = twin.topk(st, 8, table)
    assert torch.equal(v.view(torch.int32), v2.view(torch.int32)) and torch.equal(i, i2)
    assert (rk == 3).all()


# ----------------------------------------------------------------------------- 6. end to end on a DeviceFrameFeed
def test_end_to_end_actor_search_critic_on_a_feed():
    rng = np.random.default_rng(4)
    F, n_users, items, dim = 4, 60, 400, 16
    lengths = rng.integers(F + 1, 40, n_users)
    hist = [rng.integers(0, 120, n) for n in lengths]
    rat = [rng.integers(1, 6, n).astype(np.float32) for n in lengths]
    csr = HistoryCSR(np.arange(n_users), hist, rat, F)
    feed = DeviceFrameFeed(csr, torch.from_numpy(rng.normal(0, 1, (items, dim)).astype(np.float32)), DEV)
    torch.manual_seed(2)
    S = F * dim + F
    actor = recnn_b200.nn.Actor(S, dim, 32).to(DEV).eval()
    critic = recnn_b200.nn.Critic(S, dim, 32).to(DEV).eval()
    with torch.no_grad():
        critic.linear3.weight.uniform_(-0.3, 0.3)
    index = ItemIndex(feed.table, "L2")
    seen = feed.seen_items()
    pos = np.arange(n_users)
    pos_t = torch.from_numpy(pos).to(DEV)
    s = feed.user_states(pos)
    cand = index.search(actor(s), topk=64, exclude=seen, exclude_rows=pos_t).id()
    q, ids = critic.topk(s, 10, index.table, candidates=cand, exclude=seen, exclude_rows=pos_t)
    for r, u in enumerate(pos):
        got = [x for x in ids[r].tolist() if x >= 0]
        assert got and set(got) <= set(cand[r].tolist()) and not set(got) & set(hist[u].tolist())
    h = feed.holdout(pos)
    cand_h = index.search(actor(h["state"]), topk=64).id()
    rk = critic.rank(h["state"], h["target"], index.table, candidates=cand_h, exclude=seen,
                     exclude_rows=h["exclude_rows"])
    met = ranking_metrics(rk, ks=(1, 5, 10))
    assert met["n"] == n_users
    tg = h["target"].cpu().numpy()
    rest = ItemSets.from_lists([sorted(set(hist[u].tolist()) - {int(tg[r])}) for r, u in enumerate(pos)], device=DEV)
    _, i64 = critic.topk(h["state"], 64, index.table, candidates=cand_h, exclude=rest)
    check_rank_consistency(rk, i64, tg, "feed", cand_h.cpu().numpy())
    assert any(tg[r] in set(cand_h[r].tolist()) for r in range(n_users))       # some held-out items are candidates


# ----------------------------------------------------------------------------- 7. scale
def _peak_above(fn):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    out = fn()
    torch.cuda.synchronize()
    return out, torch.cuda.max_memory_allocated() - base


def test_million_items_and_all_items_memory():
    from recnn_b200 import _lib
    L = _lib.lib()
    S, A, H, I, N, M = 2570, 256, 256, 1 << 20, 2048, 1024
    torch.manual_seed(5)
    c = recnn_b200.nn.Critic(S, A, H)
    with torch.no_grad():
        c.linear3.weight.uniform_(-0.3, 0.3)
    c = c.to(DEV).eval()
    param_arena(c)
    st = torch.randn(N, S, device=DEV)
    table = torch.randn(I, A, device=DEV)
    base = torch.randint(0, I, (N, 1), device=DEV)
    cand = (base + torch.arange(M, device=DEV) * 977) % I                   # distinct within a row
    (v, i), peak = _peak_above(lambda: c.topk(st, 10, table, candidates=cand))
    ws = L.recnn_critic_serve_workspace_bytes(c.dims, N, M, I, 10, 0)
    assert peak <= ws + 2 * N * 10 * 8 + (1 << 20), (peak, ws)
    p = O.params64(c)
    for r in (0, 1000, N - 1):
        cols = cand[r:r + 1].cpu().numpy()
        q64 = O.q_pairs(p, st[r:r + 1].double().cpu().numpy(), table[cand[r]].double().cpu().numpy(),
                        np.arange(M)[None])
        check_against_float64_one(v[r], i[r], q64[0], cols[0])
    # every item: the peak does not depend on the table's size
    st64 = st[:64].contiguous()
    peaks = []
    for n_items in (131072, 262144):
        tb = table[:n_items]
        _, pk = _peak_above(lambda: c.topk(st64, 10, tb))
        peaks.append(pk)
    assert peaks[0] == peaks[1], peaks


def check_against_float64_one(v, i, q64_row, cols_row):
    check_against_float64(v[None], i[None], q64_row[None], cols_row[None], v.numel())
