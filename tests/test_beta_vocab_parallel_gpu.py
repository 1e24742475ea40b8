"""The behaviour policy beta sharded over the item vocabulary (recnn_beta_shard_*) on the GPU.

As for the sharded policy (test_reinforce_vocab_parallel_gpu.py), W > 1 runs as VIRTUAL ranks on one device
(tests/_ranks.py): W copies of the sharded Beta's public API in one process, each all-gather delivering the ranks'
records in rank order (what recnn_comm_allgather delivers).  The transport and the Python API also run at world 1;
W > 1 processes need W GPUs."""
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
from recnn_b200.nn.arena import param_arena, grad_arena
from recnn_b200.nn.update import reinforce as RF
from oracle import beta_oracle as B
from oracle import reinforce_oracle as RO
from tests._ranks import bits, chunked, one_rank_group, returned, run_ranks, shard, spawn  # noqa: F401
from tests.test_beta_gpu import REORDER_BAR, make_beta, onehot

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
L = _lib.lib()
# (S, items, rows, chunk): S % 4 != 0 (re-pitched state image kept from begin) and S % 4 == 0 (state read in place);
# local blocks chunked with a ragged last chunk (W = 2, 3) and narrower than one chunk (W = 8)
SHAPES = [(37, 1003, 33, 128), (52, 2000, 40, 256)]


def _t(x):
    return torch.from_numpy(np.ascontiguousarray(x)).to(DEV)


def _radam_beta(w, b):
    beta = make_beta(w, b)
    beta.optim = recnn_b200.optim.RAdam(beta.net.parameters(), lr=1e-2, weight_decay=1e-5)
    return beta


def _state_of(m):
    return {"p": param_arena(m).clone(), "g": grad_arena(m).clone(), "m": m.optim._m.clone(), "v": m.optim._v.clone(),
            "t": int(m.optim._t.item())}


def sharded_calls(full, world, calls, chunk=None, order=None):
    """On W virtual ranks, a Beta sharded from ``full`` is called on each (state, ids) of ``calls``: per rank, per call
    (column block or the call's exception, loss, arenas after the call, net.0's {w, b, gw, gb} after the call)."""
    def rank(r):
        beta = shard({}, full)[1]
        out = []
        for s, ids in calls:
            try:
                got = beta(s, ids)
            except (RuntimeError, IndexError) as exc:
                got = exc
            lin = beta.net[0]
            out.append((got, beta.last_loss.clone(), _state_of(beta),
                        {"w": lin.weight.detach().clone(), "b": lin.bias.detach().clone(),
                         "gw": lin.weight.grad.clone(), "gb": lin.bias.grad.clone()}))
        return out
    with chunked(calls[0][0].shape[0], chunk):
        return run_ranks(world, rank, order=order)


def _case(S, items, n, seed, world):
    rng = np.random.default_rng(seed)
    bound = 1.0 / np.sqrt(S)
    w = rng.uniform(-bound, bound, (items, S)).astype(np.float32)
    b = rng.uniform(-bound, bound, items).astype(np.float32)
    ids = rng.integers(0, items, n)
    edges = sorted({e for r in range(world) for lo, hi in [D.vocab_shard(items, r, world)]
                    for e in (lo - 1, lo, hi - 1) if 0 <= e < items})
    ids[:len(edges)] = edges[:n]
    return rng, w, b, ids


def _rel(got, want):
    return float((got - want).abs().max() / want.abs().max())


def run_virtual_sweep():
    """Every shape x W: two calls each; the loss has the same bits on every rank; the concatenated blocks, dW, db and
    the stepped weights against the unsharded Beta (reordering bar) and the float64 oracle."""
    for S, items, n, chunk in SHAPES:
        for world in (2, 3, 8):
            rng, w, b, ids = _case(S, items, n, S + items + world, world)
            full = _radam_beta(w, b)
            params, o = {"w": w.copy(), "b": b.copy()}, B.make_radam(lr=1e-2)
            it = _t(ids)
            calls = [(_t(rng.normal(0, 1, (n, S)).astype(np.float32)), it) for _ in range(2)]
            res = returned(sharded_calls(full, world, calls, chunk))
            for t, (s, _) in enumerate(calls):
                prev = {k: getattr(full.net[0], k).detach().clone() for k in ("weight", "bias")}
                with chunked(n, chunk):
                    want = full(s, it)
                got = [x[t] for x in res]
                assert not any(isinstance(g[0], Exception) for g in got), got
                assert len({bits(g[1]).item() for g in got}) == 1
                loss = float(got[0][1])
                assert loss == pytest.approx(float(full.last_loss), rel=1e-6)
                probs = torch.cat([g[0] for g in got], 1)
                assert _rel(probs, want) <= REORDER_BAR
                wp, wl, grads = B.beta_call(params, o, s.cpu().numpy(), ids)
                assert abs(loss - wl) <= 1e-5 * (abs(wl) + 0.1)
                assert np.max(np.abs(probs.double().cpu().numpy() - wp) / (wp + 1e-2 * wp.max())) <= 1e-5
                local = [g[3] for g in got]
                gw = torch.cat([x["gw"] for x in local])
                gb = torch.cat([x["gb"] for x in local])
                assert _rel(gw, full.net[0].weight.grad) <= REORDER_BAR, (S, items, world, t)
                assert _rel(gb, full.net[0].bias.grad) <= REORDER_BAR, (S, items, world, t)
                for g, k in ((gw, "w"), (gb, "b")):
                    ref = grads[k]
                    assert np.abs(g.double().cpu().numpy() - ref).max() <= 1e-4 * np.abs(ref).max(), k
                # the stepped weights: two roundings of the weight plus the gradients' reordering share of the step
                for k, key in (("weight", "w"), ("bias", "b")):
                    g = torch.cat([x[key] for x in local])
                    ref = getattr(full.net[0], k).detach()
                    tol = 2 * torch.finfo(torch.float32).eps * ref.abs() + REORDER_BAR * float((ref - prev[k]).abs().max())
                    assert bool(((g - ref).abs() <= tol).all()), k
                assert all(g[2]["t"] == t + 1 for g in got)
            print("virtual beta S %d I %d W %d: ok" % (S, items, world))


def test_virtual_ranks_against_the_unsharded_step_and_the_oracle():
    run_virtual_sweep()


def test_virtual_ranks_on_the_cuda_core_back_end():
    """The same sweep with every GEMM on the exact-fp32 CUDA-core kernel, in a process of its own (the back end is fixed
    per process)."""
    code = "import sys; sys.path.insert(0, %r); from tests import test_beta_vocab_parallel_gpu as T; " \
           "T.run_virtual_sweep()" % ROOT
    env = dict(os.environ, RECNN_B200_MATH="simt")
    r = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, cwd=ROOT)
    print(r.stdout[-3000:], r.stderr[-3000:])
    assert r.returncode == 0


@pytest.mark.parametrize("S,items,n,chunk", SHAPES)
def test_world1_is_bit_identical_to_the_step(S, items, n, chunk):
    rng, w, b, ids = _case(S, items, n, 3 * S, 1)
    full = _radam_beta(w, b)
    calls = [(_t(rng.normal(0, 1, (n, S)).astype(np.float32)), _t(rng.integers(0, items, n))) for _ in range(3)]
    (res,) = returned(sharded_calls(full, 1, calls, chunk))
    for t, ((s, it), (probs, loss, state, _)) in enumerate(zip(calls, res)):
        with chunked(n, chunk):
            want = full(s, it)
        assert torch.equal(probs, want)
        assert bits(loss).item() == bits(full.last_loss).item()
        e = _state_of(full)
        for k in state:
            assert (state[k] == e[k]) if k == "t" else torch.equal(state[k], e[k]), (t, k)


def test_records_out_of_rank_order_and_bad_ids_skip_the_step():
    S, items, n, chunk = 37, 1003, 33, 128
    rng, w, b, ids = _case(S, items, n, 5, 3)
    s = _t(rng.normal(0, 1, (n, S)).astype(np.float32))
    bad = [ids.copy(), ids.copy()]
    bad[0][7], bad[1][7] = items, -1
    # call 0 is good; the first gather of call 1 and the second of call 2 come out of rank order; calls 3 and 4 hold
    # an id out of range
    calls = [(s, _t(x)) for x in (ids, ids, ids, bad[0], bad[1])]
    res = returned(sharded_calls(_radam_beta(w, b), 3, calls, chunk, order={2: [1, 0, 2], 5: [0, 2, 1]}))
    for c, want in ((1, RuntimeError), (2, RuntimeError), (3, IndexError), (4, IndexError)):
        errs = [x[c][0] for x in res]
        assert all(isinstance(e, want) for e in errs), (c, errs)
        if want is RuntimeError:
            assert all("disagree on the vocabulary shard plan" in str(e) for e in errs)
        else:
            assert len({bits(x[c][1]).item() for x in res}) == 1
        for x in res:
            before, after = x[0][2], x[c][2]
            for k in ("p", "m", "v", "t"):
                assert (before[k] == after[k]) if k == "t" else torch.equal(before[k], after[k]), (c, k)


def test_sharded_draws_pick_the_unsharded_item():
    """W = 3: DiscreteActor.pi_beta_sample with a Beta sharded with the policy, the action drawn from beta (the
    {pi: beta, beta: beta} source): the draw from beta's blocks and records, from replayed uniforms, against the
    unsharded policy's draw on the unsharded probabilities, and pi's log-prob of it from the policy's blocks."""
    S, items, n = 37, 1003, 300
    rng, w, b, ids = _case(S, items, n, 8, 3)
    w = (w * 6).astype(np.float32)
    s = _t(rng.normal(0, 1, (n, S)).astype(np.float32))
    u = _t(rng.random(n).astype(np.float32))
    full = make_beta(w, b)
    policy = recnn_b200.nn.DiscreteActor(S, items, 16).to(DEV)

    def rank(r):
        nets, beta = shard({"policy_net": policy}, full)
        pol = nets["policy_net"]
        pol.uniform_source = lambda n: u
        pol.action_source = {"pi": "beta", "beta": "beta"}
        pi_lp, beta_lp, _ = pol.pi_beta_sample(s, beta, _t(ids))
        return pol._last_sample["action"], beta_lp, pi_lp
    with chunked(n, 128):
        res = returned(run_ranks(3, rank))
        want = full(s, _t(ids))
    a, lp, pi_lp = res[0]
    for x in res[1:]:
        assert torch.equal(x[0], a) and torch.equal(x[1], lp) and torch.equal(x[2], pi_lp)
    policy.uniform_source = lambda n: u
    ra, rl = policy._sample(want)
    _, _, margin = RO.categorical_sample(want.double().cpu().numpy(), u.cpu().numpy())
    keep = torch.from_numpy(margin > 1e-5).to(DEV)
    assert int(keep.sum()) > 0.9 * n
    assert torch.equal(a[keep], ra[keep])
    assert float((lp[keep] - rl[keep]).abs().max()) <= 1e-5
    want_pi = RO.categorical_log_prob(policy(s).double().cpu().numpy(), a.cpu().numpy())
    assert np.abs(pi_lp.cpu().numpy() - want_pi).max() <= 1e-5


class Call:
    """The args of one Beta's call on its own arena (built-in RAdam, or external), with its own workspace: the rank
    share memory test runs the C phases itself."""

    def __init__(self, beta, state, ids, chunk):
        d = beta.dims
        n = state.shape[0]
        self.chunk = chunk if chunk < d.num_items else d.num_items
        self.probs = torch.empty(n, d.num_items, device=DEV)
        self.loss = torch.empty((), device=DEV)
        self.error = torch.zeros(1, dtype=torch.int32, device=DEV)
        self.ws = torch.empty(L.recnn_beta_workspace_bytes(d, n, self.chunk), dtype=torch.uint8, device=DEV)
        a = _lib.BetaArgs()
        a.dims, a.n_rows, a.chunk_items = d, n, self.chunk
        a.net, a.optim = beta.optim.c_net(beta), beta.optim.c_optim()
        a.state, a.state_ld = state.data_ptr(), state.stride(0)
        a.action, a.probs_out = ids.data_ptr(), self.probs.data_ptr()
        a.loss, a.error = self.loss.data_ptr(), self.error.data_ptr()
        a.workspace, a.workspace_bytes = self.ws.data_ptr(), self.ws.numel()
        self.args = a


# ----------------------------------------------------------------------------- the Python API at world 1
def _notebook_agent(source, items=1003, H=64, S=37):
    torch.manual_seed(9)
    beta_net = recnn_b200.nn.Beta(S, items).to(DEV)
    value_net = recnn_b200.nn.Critic(S, items, H, 54e-2).to(DEV)
    policy_net = recnn_b200.nn.DiscreteActor(S, items, H).to(DEV)
    policy_net.action_source = source
    reinforce = recnn_b200.nn.Reinforce(policy_net, value_net).to(torch.device(DEV))
    seen = []

    def beta_forward(state, action):
        p = beta_net.forward(state, action)
        seen.append(p.clone())
        return p

    def select_action_corr(state, action, K, writer, step, **kwargs):
        return reinforce.nets["policy_net"]._select_action_with_TopK_correction(state, beta_forward, action, K=K,
                                                                               writer=writer, step=step)

    reinforce.nets["policy_net"].select_action = select_action_corr
    reinforce.params["reinforce"] = recnn_b200.nn.ChooseREINFORCE(
        recnn_b200.nn.ChooseREINFORCE.reinforce_with_TopK_correction)
    reinforce.params["K"] = 10
    return reinforce, beta_net, seen


@pytest.mark.parametrize("source", [{"pi": "pi", "beta": "beta"}, {"pi": "beta", "beta": "beta"}],
                         ids=["pi_pi", "pi_beta"])
def test_python_api_world1_equals_unsharded(one_rank_group, source):
    S, items, N, steps = 37, 1003, 10, 11
    plain, plain_beta, plain_seen = _notebook_agent(source)
    shard, shard_beta, shard_seen = _notebook_agent(source)
    D.enable_vocab_parallel(shard, beta=shard_beta)
    vp = shard.nets["policy_net"].__dict__["_recnn_vp"]
    assert shard_beta.__dict__["_recnn_vp"] is vp and (vp.lo, vp.hi, vp.world) == (0, items, 1)
    rng = np.random.default_rng(4)
    for step in range(steps):
        ids = rng.integers(0, items, N)
        b = {"state": torch.from_numpy(rng.normal(0, 1, (N, S)).astype(np.float32)), "action": torch.from_numpy(ids),
             "reward": torch.from_numpy(rng.integers(1, 6, N).astype(np.float32) - 3),
             "next_state": torch.from_numpy(rng.normal(0, 1, (N, S)).astype(np.float32)),
             "done": torch.from_numpy((rng.random(N) < 0.1).astype(np.float32))}
        losses = []
        for agent in (plain, shard):
            torch.manual_seed(1000 + step)         # the same dropout masks and draws for both agents
            losses.append(agent.update(dict(b)))
        for agent in (plain, shard):
            agent.step()
        assert losses[0] == losses[1], step
        assert torch.equal(plain_seen[-1], shard_seen[-1]), step
        assert bits(plain_beta.last_loss).tolist() == bits(shard_beta.last_loss).tolist()
        pp, sp = plain.nets["policy_net"], shard.nets["policy_net"]
        for k in ("saved_log_probs", "correction", "lambda_k"):
            assert len(getattr(pp, k)) == len(getattr(sp, k))
            for x, y in zip(getattr(pp, k), getattr(sp, k)):
                if source["pi"] == "pi":
                    assert torch.equal(x, y), (step, k)
                else:
                    # pi's log-prob of beta's draw: a sharded policy reads p[a] of its block (the softmax sums to 1
                    # over all ranks), the unsharded one divides by the row's fp32 sum, as torch's Categorical does
                    torch.testing.assert_close(x, y, rtol=1e-5, atol=1e-6)
    assert plain_beta.optim.steps_taken() == shard_beta.optim.steps_taken() == steps
    for x, y in ((plain_beta, shard_beta), (plain.nets["policy_net"], shard.nets["policy_net"]),
                 (plain.nets["value_net"], shard.nets["value_net"])):
        assert torch.equal(bits(param_arena(x)), bits(param_arena(y)))
    assert torch.equal(plain_beta.optim._m, shard_beta.optim._m) and torch.equal(plain_beta.optim._v, shard_beta.optim._v)
    # one-hot and item-id actions drive the sharded beta identically
    s = torch.randn(N, S, device=DEV)
    ids = torch.randint(0, items, (N,), device=DEV)
    t0 = shard_beta.optim.steps_taken()
    p1 = shard_beta(s, onehot(ids, items))
    p2 = plain_beta(s, onehot(ids, items))
    assert torch.equal(p1, p2) and shard_beta.optim.steps_taken() == t0 + 1
    # error paths of a sharded beta
    bad = ids.clone()
    bad[2] = items
    with pytest.raises(IndexError):
        shard_beta(s, bad)
    assert shard_beta.optim.steps_taken() == t0 + 1
    pol = shard.nets["policy_net"]
    with pytest.raises(ValueError, match="not vocabulary-parallel"):
        plain.nets["policy_net"].pi_beta_sample(s, lambda st, action=None: shard_beta(st, ids), ids)
    other = D.VocabParallel(0, items, items, vp.group, 0, 2, vp.comm)
    pol.__dict__["_recnn_vp"] = other
    try:
        with pytest.raises(ValueError, match="sharded on"):
            pol.pi_beta_sample(s, lambda st, action=None: shard_beta(st, ids), ids)
    finally:
        pol.__dict__["_recnn_vp"] = vp
    with pytest.raises(RuntimeError, match="already"):
        D.enable_vocab_parallel(recnn_b200.nn.DiscreteActor(S, items, 64).to(DEV), beta=shard_beta)
    vp.comm.close()


# ----------------------------------------------------------------------------- one rank's share of the target config
def rank_share_memory():
    """S 2570, 2^20 items over 8 ranks (131,072 local), 2,048 rows, built-in RAdam: begin / rows / end of the last
    rank with the other ranks' records standing in as copies of this one's (headers fixed up)."""
    S, items, world, n = 2570, 1 << 20, 8, 2048
    rank = world - 1
    lo, hi = D.vocab_shard(items, rank, world)
    torch.manual_seed(3)
    with torch.device(DEV):
        beta = recnn_b200.nn.Beta(S, hi - lo)
        state = torch.randn(n, S)
        ids = torch.randint(0, items, (n,))
    beta.optim.c_net(beta)                       # the four arenas exist before the measurement
    d = beta.dims
    chunk = RF._chunk_items(n, d.num_items)
    vs = _lib.VocabShard(lo, items, rank, world)
    nrec = L.recnn_vocab_record_floats(n)
    gc.collect()
    torch.cuda.synchronize()
    resident = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    c = Call(beta, state, ids, chunk)
    rec = torch.empty(nrec, device=DEV)

    def gathered(x):
        g = x.repeat(world)
        hdr = g.view(world, -1)[:, :2].view(torch.int32)
        for q in range(world):
            hdr[q] = torch.tensor(D.vocab_shard(items, q, world), dtype=torch.int32)
        return g

    st = _lib.stream_ptr()
    _lib.check(L.recnn_beta_shard_begin(c.args, vs, rec.data_ptr(), st))
    g1 = gathered(rec)
    sums = torch.empty_like(rec)
    _lib.check(L.recnn_beta_shard_rows(c.args, vs, g1.data_ptr(), sums.data_ptr(), st))
    _lib.check(L.recnn_beta_shard_end(c.args, vs, gathered(sums).data_ptr(), st))
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - resident
    total = torch.cuda.max_memory_allocated()
    bound = c.ws.numel() + c.probs.numel() * 4 + (2 * world + 2) * nrec * 4
    print("beta rank share: chunk %d, workspace %.2f GB, block %.2f GB, peak above the arenas %.2f GB, total %.2f GB"
          % (chunk, c.ws.numel() / 1e9, c.probs.numel() * 4 / 1e9, peak / 1e9, total / 1e9))
    assert int(c.error) == 0 and np.isfinite(float(c.loss))
    assert beta.optim.steps_taken() == 1
    assert peak <= bound + (16 << 20)
    assert total < 12e9                  # the unsharded call holds 54.2 GB


def test_target_config_rank_share_memory():
    code = "import sys; sys.path.insert(0, %r); from tests import test_beta_vocab_parallel_gpu as T; " \
           "T.rank_share_memory()" % ROOT
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, cwd=ROOT)
    print(r.stdout[-2000:], r.stderr[-2000:])
    assert r.returncode == 0


# ----------------------------------------------------------------------------- W > 1 processes
def _case_np(world):
    return _case(37, 1003, 24, 77, world)


def _vp_worker(rank, world, port, q):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    try:
        rng, w, b, ids = _case_np(world)
        state = rng.normal(0, 1, (24, 37)).astype(np.float32)
        beta = recnn_b200.nn.Beta(37, 1003)
        if rank == 0:
            beta.load_state_dict({"net.0.weight": torch.from_numpy(w), "net.0.bias": torch.from_numpy(b)})
        beta = beta.to(dev)
        policy = recnn_b200.nn.DiscreteActor(37, 1003, 16).to(dev)
        D.enable_vocab_parallel(policy, beta=beta)
        block = beta(torch.from_numpy(state).to(dev), torch.from_numpy(ids).to(dev))
        vp = beta.__dict__["_recnn_vp"]
        q.put((rank, {"loss": float(beta.last_loss), "lo": vp.lo, "hi": vp.hi, "block": block.cpu().numpy(),
                      "gw": beta.net[0].weight.grad.cpu().numpy(), "gb": beta.net[0].bias.grad.cpu().numpy()}))
        torch.cuda.synchronize()
        vp.comm.close()
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 4, 8])
def test_multi_process_equals_unsharded(world):
    if torch.cuda.device_count() < world:
        pytest.skip("needs %d GPUs" % world)
    res = dict(spawn(_vp_worker, world))
    rng, w, b, ids = _case_np(world)
    state = rng.normal(0, 1, (24, 37)).astype(np.float32)
    full = make_beta(w, b)
    want = full(_t(state), _t(ids))
    for r in range(world):
        assert res[r]["loss"] == res[0]["loss"]
    assert res[0]["loss"] == pytest.approx(float(full.last_loss), rel=1e-6)
    for k, ref in (("block", want), ("gw", full.net[0].weight.grad), ("gb", full.net[0].bias.grad)):
        got = torch.from_numpy(np.concatenate([res[r][k] for r in range(world)], 1 if k == "block" else 0))
        assert _rel(got, ref.cpu()) <= REORDER_BAR, k
