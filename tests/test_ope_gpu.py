"""Off-policy estimation on the GPU: DiscreteActor.log_prob and Beta.log_prob against float64 at unaligned shapes and
forced chunkings on both GEMM back ends, pi's against rank()'s bits, beta's against the probabilities Beta.forward
returns, the nets' state left alone, virtual vocabulary ranks (tests/_ranks.py) and data-parallel replicas, 1M items
with bounded memory, the feed's held-out reward, and an end-to-end estimate whose answer is known."""
from __future__ import annotations

import gc
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import recnn_b200
from recnn_b200 import _lib
from recnn_b200 import dist as D
from recnn_b200.data import DeviceFrameFeed, HistoryCSR
from recnn_b200.nn.arena import param_arena
from recnn_b200.nn.update.reinforce import _chunk_items
from recnn_b200.utils.metrics import off_policy_estimates
from tests import _ope_oracle as O
from tests._discrete import make_policy
from tests._ranks import _copy, bits, chunked, exchange, returned, run_ranks, shard
from tests.test_beta_gpu import make_beta, onehot, snapshot
from tests.test_policy_topk_gpu import SHAPES, Z_BAR, make_case
from tests import _policy_topk_oracle as TK

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
L = _lib.lib()


def _t(x):
    return torch.from_numpy(np.ascontiguousarray(x)).to(DEV)


def beta_case(S, I, seed, spread=4.0):
    rng = np.random.default_rng(seed)
    w = (rng.normal(0, spread / np.sqrt(S), (I, S))).astype(np.float32)
    b = rng.normal(0, 0.5, I).astype(np.float32)
    return w, b


def edge_actions(rng, n, items, cuts=()):
    """Random ids with 0, items - 1, the 128- and 256-chunk edges and ``cuts`` +-1 in the first rows."""
    a = rng.integers(0, items, n)
    edges = sorted({e for c in (0, 128, 256, items) + tuple(cuts) for e in (c - 1, c) if 0 <= e < items})
    a[:len(edges)] = edges[:n]
    return a.astype(np.int64)


def check_close(got, want, z, what):
    err = np.abs(got.cpu().numpy().astype(np.float64) - want)
    assert err.max() <= 4 * Z_BAR * (1 + np.abs(z).max()), (what, err.max())


# ----------------------------------------------------------------------------- 1. float64, both back ends
def run_sweep():
    for S, H, I, N in SHAPES:
        p, state = make_case(S, H, I, N, 3 * S + I)
        m = make_policy(p, S, H, I)
        w, b = beta_case(S, I, S + I)
        beta = make_beta(w, b)
        st = _t(state)
        a = edge_actions(np.random.default_rng(I), N, I)
        ad = _t(a)
        z_pi = TK.logits(p, state)
        z_b = state.astype(np.float64) @ w.astype(np.float64).T + b
        want_pi = O.policy_log_prob(p["w1"], p["b1"], p["w2"], p["b2"], state, a)
        want_b = O.beta_log_prob(w, b, state, a)
        for chunk in (None, 128, 256):
            with chunked(N, chunk):
                lp = m.log_prob(st, ad)
                _, lr = m.rank(st, ad)
                lb = beta.log_prob(st, ad)
                lb1 = beta.log_prob(st, onehot(ad, I))
            check_close(lp, want_pi, z_pi, ("pi", S, I, chunk))
            assert torch.equal(bits(lp), bits(lr)), ("pi == rank", S, I, chunk)
            check_close(lb, want_b, z_b, ("beta", S, I, chunk))
            assert torch.equal(bits(lb), bits(lb1)), ("one-hot == ids", S, I, chunk)
        print("log_prob S %d I %d N %d: ok" % (S, I, N))


def test_against_float64_and_rank():
    run_sweep()


def test_against_float64_on_the_cuda_core_back_end():
    code = "import sys; sys.path.insert(0, %r); from tests import test_ope_gpu as T; T.run_sweep()" % ROOT
    env = dict(os.environ, RECNN_B200_MATH="simt")
    r = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, cwd=ROOT)
    print(r.stdout[-3000:], r.stderr[-3000:])
    assert r.returncode == 0


def test_beta_log_prob_is_the_log_of_forwards_probabilities():
    """Beta.forward returns the probabilities from before its step; on a copy, their log at the action is what
    log_prob gives (up to the rounding of log(exp(z - M) / S) against z - M - log S)."""
    S, I, N = 37, 1003, 33
    w, b = beta_case(S, I, 5)
    beta = make_beta(w, b)
    state = torch.randn(N, S, device=DEV)
    a = _t(edge_actions(np.random.default_rng(5), N, I))
    for chunk in (None, 128):
        with chunked(N, chunk):
            lp = beta.log_prob(state, a)
            probs = _copy(beta)(state, a)
        want = torch.log(probs[torch.arange(N, device=DEV), a].double())
        assert float((lp.double() - want).abs().max()) <= 2e-6 * (1 + float(want.abs().max())), chunk


def test_out_of_range_ids_raise():
    S, H, I, N = 20, 16, 300, 8
    p, state = make_case(S, H, I, N, 9)
    m = make_policy(p, S, H, I)
    beta = make_beta(*beta_case(S, I, 9))
    st = _t(state)
    for bad in (I, -1):
        a = torch.arange(N, device=DEV)
        a[3] = bad
        with pytest.raises(IndexError):
            m.log_prob(st, a)
        with pytest.raises(IndexError):
            beta.log_prob(st, a)
    assert m.log_prob(st[:0], torch.zeros(0, dtype=torch.int64)).shape == (0,)
    assert beta.log_prob(st[:0], torch.zeros(0, dtype=torch.int64)).shape == (0,)


# ----------------------------------------------------------------------------- 2. the nets' state
def test_log_prob_leaves_the_nets_state_alone():
    S, H, I, N = 20, 16, 300, 8
    p, state = make_case(S, H, I, N, 9)
    m = make_policy(p, S, H, I)
    st = _t(state)
    m.select_action(st)
    saved = (len(m.saved_log_probs), len(m._saved), m._draws)
    snap = [dict(x) for x in m._saved]
    logp0 = m.saved_log_probs[0].clone()
    arena = param_arena(m).clone()
    lp = m.log_prob(st, m._saved[0]["action"])
    assert (len(m.saved_log_probs), len(m._saved), m._draws) == saved
    assert torch.equal(m.saved_log_probs[0], logp0) and torch.equal(param_arena(m), arena)
    assert all(torch.equal(x["state"], y["state"]) and torch.equal(x["action"], y["action"])
               for x, y in zip(m._saved, snap))
    assert torch.allclose(lp, logp0, atol=1e-4)           # the sampler's log-prob, within the Categorical clamp

    beta = make_beta(*beta_case(S, I, 10))
    a = m._saved[0]["action"]
    beta(st, a)                                            # a step: last_loss, gradients and RAdam state exist
    before = snapshot(beta)
    loss = beta.last_loss
    loss_bits = bits(loss.reshape(1)).clone()
    beta.log_prob(st, a)
    beta.log_prob(st, onehot(a, I))
    after = snapshot(beta)
    assert beta.last_loss is loss and torch.equal(bits(beta.last_loss.reshape(1)), loss_bits)
    for k in before:
        assert np.array_equal(np.asarray(before[k]), np.asarray(after[k])), k
    assert "_recnn_block" not in beta.__dict__


# ----------------------------------------------------------------------------- 3. virtual vocabulary ranks
def sharded_log_probs(full, beta, world, state, action, chunk=None, order=None, block=False):
    def rank(r):
        nets, b = shard({"policy_net": full}, beta)
        pol = nets["policy_net"]
        held = None
        if block:
            b(state, action)                               # a sharded step registers its block
            held = b.__dict__["_recnn_block"]
        out = (pol.log_prob(state, action), b.log_prob(state, action))
        if block:
            assert b.__dict__["_recnn_block"] is held
        return out
    with chunked(state.shape[0], chunk):
        return run_ranks(world, rank, order=order)


@pytest.mark.parametrize("world", [1, 2, 3, 8])
def test_virtual_ranks(world):
    S, H, I, N = 52, 64, 1003, 40
    p, state = make_case(S, H, I, N, world + 30)
    full = make_policy(p, S, H, I)
    w, b = beta_case(S, I, world + 31)
    beta = make_beta(w, b)
    st = _t(state)
    cuts = [lo for lo, _ in TK.item_plan(I, world)][1:]
    a = edge_actions(np.random.default_rng(world), N, I, cuts)
    ad = _t(a)
    want_pi = O.policy_log_prob(p["w1"], p["b1"], p["w2"], p["b2"], state, a)
    want_b = O.beta_log_prob(w, b, state, a)
    for chunk in (None, 128):
        res = returned(sharded_log_probs(full, beta, world, st, ad, chunk, block=chunk is None))
        lp, lb = res[0]
        for x in res[1:]:
            assert torch.equal(bits(x[0]), bits(lp)) and torch.equal(bits(x[1]), bits(lb)), ("W", world, chunk)
        check_close(lp, want_pi, TK.logits(p, state), ("pi W", world, chunk))
        check_close(lb, want_b, state.astype(np.float64) @ w.astype(np.float64).T + b, ("beta W", world, chunk))
        if world == 1:
            with chunked(N, chunk):
                assert torch.equal(bits(full.log_prob(st, ad)), bits(lp))
                assert torch.equal(bits(beta.log_prob(st, ad)), bits(lb))
    if world > 1:
        res = sharded_log_probs(full, beta, world, st, ad, order={0: [1, 0] + list(range(2, world))})
        assert all(isinstance(e, RuntimeError) and "disagree on the vocabulary shard plan" in str(e)
                   for e in res), res
    res = sharded_log_probs(full, beta, world, st, _t(np.where(np.arange(N) == 2, I, a)))
    assert all(isinstance(e, IndexError) for e in res), res


# ----------------------------------------------------------------------------- 4. data-parallel replicas
@pytest.mark.parametrize("world", [2, 3])
def test_data_parallel_replicas_stay_local(world):
    S, H, I, N = 37, 32, 2000, 61
    p, state = make_case(S, H, I, N, 50 + world)
    full = make_policy(p, S, H, I)
    beta = make_beta(*beta_case(S, I, 51 + world))
    st = _t(state)
    a = _t(edge_actions(np.random.default_rng(world), N, I))
    cuts = np.sort(np.random.default_rng(world).choice(np.arange(1, N), world - 1, replace=False))
    bounds = list(zip([0] + cuts.tolist(), cuts.tolist() + [N]))

    def rank(r):
        m, b = _copy(full), _copy(beta)
        ex = exchange()
        D.data_parallel_in_place({"policy_net": m}, D.RowParallel(None, ex.rank, ex.world, ex), b)
        lo, hi = bounds[r]
        return m.log_prob(st[lo:hi], a[lo:hi]), b.log_prob(st[lo:hi], a[lo:hi])
    log = []
    res = returned(run_ranks(world, rank, log=log))
    assert log == []                                       # no exchange
    for r, (lo, hi) in enumerate(bounds):
        assert torch.equal(bits(res[r][0]), bits(full.log_prob(st[lo:hi], a[lo:hi])))
        assert torch.equal(bits(res[r][1]), bits(beta.log_prob(st[lo:hi], a[lo:hi])))


# ----------------------------------------------------------------------------- 5. 1M items
def _peak(fn):
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    out = fn()
    torch.cuda.synchronize()
    return out, torch.cuda.max_memory_allocated() - base


def test_million_items_memory_and_sampled_rows():
    """S 2570 / H 256, 2^20 items x 2,048 rows: each call's extra memory is its workspace plus the output (no
    [N, num_items] buffer), and sampled rows match float64."""
    S, H, I, N = 2570, 256, 1 << 20, 2048
    torch.manual_seed(0)
    st = torch.randn(N, S, device=DEV)
    a = torch.randint(0, I, (N,), device=DEV)
    rows = torch.arange(0, N, N // 16, device=DEV)
    chunk = _chunk_items(N, I)

    gc.collect()                     # nets of earlier tests (module <-> optimizer cycles) hold device memory until then
    torch.cuda.empty_cache()
    with torch.device(DEV):
        m = recnn_b200.nn.DiscreteActor(S, I, H)
    with torch.no_grad():
        m.linear2.weight.mul_(8.0)
    param_arena(m)
    ws = L.recnn_discrete_rank_workspace_bytes(m.dims, N, chunk)
    lp, peak = _peak(lambda: m.log_prob(st, a))
    print("1M items x %d rows: pi log_prob peak extra %.3f GB, workspace %.3f GB" % (N, peak / 1e9, ws / 1e9))
    assert peak <= ws + N * 4 + (8 << 20) and peak < N * I * 4 / 4
    with torch.no_grad():
        x = st[rows].double()
        h = torch.relu(x @ m.linear1.weight.double().T + m.linear1.bias.double())
        z = torch.cat([h @ m.linear2.weight[c:c + 65536].double().T + m.linear2.bias[c:c + 65536].double()
                       for c in range(0, I, 65536)], 1)
    want = torch.log_softmax(z, 1)[torch.arange(len(rows), device=DEV), a[rows]]
    assert float((lp[rows].double() - want).abs().max()) <= 4 * Z_BAR * (1 + float(z.abs().max()))
    del m, h, z
    gc.collect()
    torch.cuda.empty_cache()
    with torch.device(DEV):
        beta = recnn_b200.nn.Beta(S, I)
    param_arena(beta)
    ws = L.recnn_beta_log_prob_workspace_bytes(beta.dims, N, chunk)
    lb, peak = _peak(lambda: beta.log_prob(st, a))
    print("1M items x %d rows: beta log_prob peak extra %.3f GB, workspace %.3f GB" % (N, peak / 1e9, ws / 1e9))
    assert peak <= ws + N * 4 + (8 << 20) and peak < N * I * 4 / 4
    lin = beta.net[0]
    with torch.no_grad():
        x = st[rows].double()
        z = torch.cat([x @ lin.weight[c:c + 65536].double().T + lin.bias[c:c + 65536].double()
                       for c in range(0, I, 65536)], 1)
    want = torch.log_softmax(z, 1)[torch.arange(len(rows), device=DEV), a[rows]]
    assert float((lb[rows].double() - want).abs().max()) <= 4 * Z_BAR * (1 + float(z.abs().max()))


# ----------------------------------------------------------------------------- 6. the feed, end to end
def _feed(seed, F=4, n_users=60, items=300, dim=8):
    rng = np.random.default_rng(seed)
    lengths = rng.integers(F + 1, 30, n_users)
    hist = [rng.integers(0, items, n) for n in lengths]
    rat = [rng.integers(1, 6, n).astype(np.float32) for n in lengths]
    csr = HistoryCSR(np.arange(n_users), hist, rat, F)
    table = torch.from_numpy(rng.uniform(0, 1, (items, dim)).astype(np.float32))     # non-negative states
    return DeviceFrameFeed(csr, table, DEV), csr, hist, rat


def test_feed_holdout_reward():
    feed, csr, hist, rat = _feed(4)
    pos = np.arange(csr.n_users)[::-1].copy()
    h = feed.holdout(pos)
    last = csr.win_offsets[pos + 1] - 1
    e = feed.embed(feed.windows(last))
    assert torch.equal(bits(h["reward"]), bits(e["reward"]))
    assert torch.equal(bits(h["state"]), bits(e["state"]))
    assert np.array_equal(h["reward"].cpu().numpy(), [rat[u][-1] for u in pos])
    assert set(h) == {"state", "target", "reward", "exclude_rows", "window_ids"}


def test_end_to_end_when_pi_equals_beta():
    """A policy whose logits are beta's (H = S, W1 = I, b1 = 0 on non-negative states, W2 / b2 = beta's): every weight
    is 1 up to rounding, so IPS is the mean logged reward and the effective sample size is n."""
    feed, csr, _, _ = _feed(8)
    h = feed.holdout(np.arange(csr.n_users))
    S = h["state"].shape[1]
    items = feed.table.shape[0]
    torch.manual_seed(3)
    beta = recnn_b200.nn.Beta(S, items).to(DEV)
    with torch.no_grad():
        beta.net[0].weight.mul_(20.0)                       # logits far from uniform
    pi = recnn_b200.nn.DiscreteActor(S, items, S).to(DEV)
    with torch.no_grad():
        pi.linear1.weight.copy_(torch.eye(S))
        pi.linear1.bias.zero_()
        pi.linear2.weight.copy_(beta.net[0].weight)
        pi.linear2.bias.copy_(beta.net[0].bias)
    lp_pi = pi.log_prob(h["state"], h["target"])
    lp_b = beta.log_prob(h["state"], h["target"])
    assert float(lp_b.std()) > 0.1
    est = off_policy_estimates(lp_pi, lp_b, h["reward"])
    r = h["reward"].double()
    assert est["logged_reward"] == pytest.approx(float(r.mean()), rel=1e-12)
    assert est["ips"] == pytest.approx(float(r.mean()), rel=1e-4)
    assert est["snips"] == pytest.approx(float(r.mean()), rel=1e-4)
    assert est["ess"] == pytest.approx(csr.n_users, rel=1e-4)
    assert est["max_weight"] == pytest.approx(1.0, rel=1e-4)
