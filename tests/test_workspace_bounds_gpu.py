"""Both sides of the workspace contract of every entry point that works in caller memory.

Each entry point sizes its workspace / scratch with a query and cuts it with the same layout function.  Here every one
of them runs on exactly the reported size, placed 16 bytes (not 256) into a larger buffer whose bytes outside that
window hold a canary: the canary must survive and the results must be the bits of a run on a fresh, generous buffer.
For the byte workspaces, one byte less must be refused with RECNN_E_WORKSPACE before anything is launched.  Every write
stays inside a live allocation: an overrun shows up as a changed canary, never as a fault."""
from __future__ import annotations

import numpy as np
import pytest
import torch

import recnn_b200
from recnn_b200 import _lib
from recnn_b200.nn.arena import param_arena, grad_arena
from recnn_b200.nn.update._engine import StepEngine, DDPG_NETS, TD3_NETS
from oracle import cases as OC
from oracle import reinforce_oracle as RO
from tests._cuda import load_net
from tests._discrete import critic_case, critic_ranks, make_policy

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
L = _lib.lib()
E_WORKSPACE = -3
CANARY = 0xA5
OFFSET = 16                 # 16-byte aligned, not 256-byte aligned
GUARD = 1 << 16             # canary bytes behind the window
# (S, H, items, rows, chunk): S % 4 == 0 with the items chunked (ragged last chunk); S % 4 != 0 and H % 4 != 0 with one
# chunk
DISCRETE = [(52, 64, 1003, 40, 128), (37, 30, 300, 33, 300)]
# (S, A, H, rows)
DENSE = [(52, 16, 64, 40), (37, 7, 30, 33)]


def _bytes(t):
    return t.detach().reshape(-1).view(torch.uint8).clone()


def check_exact_size(size, unit, run, state):
    """run(ptr, nbytes) -> the statuses of the call(s) on the workspace at ptr; state: the device tensors they write
    (restored before each run).  size: the query's answer, in units of `unit` bytes."""
    init = [t.clone() for t in state]

    def go(ptr, nbytes):
        for t, s in zip(state, init):
            t.copy_(s)
        statuses = run(ptr, nbytes)
        assert statuses and all(st == 0 for st in statuses), (statuses, L.recnn_b200_last_error())
        torch.cuda.synchronize()
        return [_bytes(t) for t in state]

    nbytes = size * unit
    fresh = torch.zeros(nbytes + GUARD, dtype=torch.uint8, device=DEV)
    want = go(fresh.data_ptr(), fresh.numel())
    buf = torch.full((OFFSET + nbytes + GUARD,), CANARY, dtype=torch.uint8, device=DEV)
    got = go(buf.data_ptr() + OFFSET, nbytes)
    assert bool((buf[:OFFSET] == CANARY).all()), "write before the workspace"
    tail = (buf[OFFSET + nbytes:] != CANARY).nonzero()
    assert tail.numel() == 0, "write %d bytes past the reported size" % (int(tail[0]) + 1)
    for i, (w, g) in enumerate(zip(want, got)):
        assert torch.equal(w, g), "output %d differs from the run on a fresh buffer" % i


def check_too_small(nbytes, run):
    """one byte less than the reported size: every call refuses it with RECNN_E_WORKSPACE and launches nothing"""
    buf = torch.zeros(nbytes, dtype=torch.uint8, device=DEV)
    before = L.recnn_b200_launch_count()
    statuses = run(buf.data_ptr(), nbytes - 1)
    assert statuses == [E_WORKSPACE] * len(statuses), statuses
    assert b"workspace too small" in L.recnn_b200_last_error()
    assert L.recnn_b200_launch_count() == before


# ---------------------------------------------------------------- the DDPG / TD3 step
def _step_case(algo, S, A, H, n):
    torch.manual_seed(S * 1000 + H)
    names = DDPG_NETS if algo == _lib.ALGO_DDPG else TD3_NETS
    nets = {k: (recnn_b200.nn.Actor(S, A, H) if "policy" in k else recnn_b200.nn.Critic(S, A, H, 3e-3)).to(DEV)
            for k in names}
    for k, m in nets.items():
        m.eval() if k.startswith("target") else m.train()       # perf-mode dropout from Philox
    opts = {"policy_optimizer": recnn_b200.optim.Adam(nets["policy_net"].parameters(), lr=1e-3)}
    for k in names:
        if k.startswith("value_net"):
            opts["value_optimizer" + k[len("value_net"):]] = recnn_b200.optim.Adam(nets[k].parameters(), lr=1e-3)
    g = torch.Generator().manual_seed(n)
    batch = {"state": torch.randn(n, S, generator=g), "next_state": torch.randn(n, S, generator=g),
             "action": torch.randn(n, A, generator=g), "reward": torch.randn(n, generator=g),
             "done": (torch.rand(n, generator=g) < 0.2).float()}
    eng = StepEngine(algo, nets, DEV)
    params = dict(OC.DDPG_PARAMS if algo == _lib.ALGO_DDPG else OC.TD3_PARAMS)
    a, _, _ = eng._build_args(eng._stage_batch(batch), nets, opts, params, True, True)
    a.phases = _lib.PH_ALL
    a.losses_host = None
    state = [eng.losses, eng.rng_step]
    for k, m in nets.items():
        state.append(param_arena(m))
        if not k.startswith("target"):
            state.append(grad_arena(m))
    for o in opts.values():
        state += [t for t in (o._m, o._v, o._t, o._slow) if t is not None]
    fn = L.recnn_ddpg_step if algo == _lib.ALGO_DDPG else L.recnn_td3_step

    def run(ptr, nbytes):
        assert eng.buf      # the engine owns the staged batch the args point into: it must outlive every call
        a.workspace, a.workspace_bytes = ptr, nbytes
        return [fn(a, _lib.stream_ptr())]
    return L.recnn_step_workspace_bytes(a.dims, n, algo), run, state


@pytest.mark.parametrize("algo", [_lib.ALGO_DDPG, _lib.ALGO_TD3])
@pytest.mark.parametrize("S,A,H,n", DENSE)
def test_step(algo, S, A, H, n):
    size, run, state = _step_case(algo, S, A, H, n)
    check_exact_size(size, 1, run, state)
    check_too_small(size, run)


# ---------------------------------------------------------------- Actor / Critic forward
@pytest.mark.parametrize("S,A,H,n", DENSE)
def test_actor_and_critic_forward(S, A, H, n):
    torch.manual_seed(S + H)
    d = _lib.Dims(S, A, H, 0)
    actor, critic = recnn_b200.nn.Actor(S, A, H).to(DEV), recnn_b200.nn.Critic(S, A, H, 3e-3).to(DEV)
    s, act = torch.randn(n, S, device=DEV), torch.randn(n, A, device=DEV)
    out_a, out_c = torch.zeros(n, A, device=DEV), torch.zeros(n, device=DEV)

    def run_actor(ptr, nbytes):
        return [L.recnn_actor_forward(d, param_arena(actor).data_ptr(), s.data_ptr(), n, None, None, 1,
                                      out_a.data_ptr(), ptr, _lib.stream_ptr())]

    def run_critic(ptr, nbytes):
        return [L.recnn_critic_forward(d, param_arena(critic).data_ptr(), s.data_ptr(), act.data_ptr(), n, None, None,
                                       out_c.data_ptr(), ptr, _lib.stream_ptr())]
    check_exact_size(L.recnn_forward_scratch_floats(d, n, 0), 4, run_actor, [out_a])
    check_exact_size(L.recnn_forward_scratch_floats(d, n, 1), 4, run_critic, [out_c])


# ---------------------------------------------------------------- the DiscreteActor: forward, policy gradient, shards
def _discrete(S, H, I, n, seed=3):
    rng = np.random.default_rng(seed)
    m = make_policy(RO.make_discrete_actor(rng, S, I, H), S, H, I)
    state = torch.from_numpy(rng.normal(0, 1, (n, S)).astype(np.float32)).to(DEV)
    action = torch.from_numpy(rng.integers(0, I, n)).to(DEV)
    ret = torch.from_numpy(rng.normal(0, 1, n).astype(np.float32)).to(DEV)
    blp = torch.from_numpy(np.log(rng.uniform(0.001, 0.01, n)).astype(np.float32)).to(DEV)
    return m, state, action, ret, blp


@pytest.mark.parametrize("S,H,I,n,chunk", DISCRETE)
def test_discrete_forward_and_policy_grad(S, H, I, n, chunk):
    m, state, action, ret, blp = _discrete(S, H, I, n)
    d, p = m.dims, param_arena(m)
    probs = torch.zeros(n, I, device=DEV)
    grads, out = torch.zeros_like(p), torch.zeros(2, device=DEV)

    def run_forward(ptr, nbytes):
        return [L.recnn_discrete_forward(d, p.data_ptr(), state.data_ptr(), n, probs.data_ptr(), ptr,
                                         _lib.stream_ptr())]

    def run_grad(ptr, nbytes):
        return [L.recnn_reinforce_policy_grad_chunked(
            d, p.data_ptr(), grads.data_ptr(), state.data_ptr(), action.data_ptr(), blp.data_ptr(), ret.data_ptr(), n,
            _lib.REINFORCE_TOPK, 4, chunk, out.data_ptr(), ptr, _lib.stream_ptr())]
    check_exact_size(L.recnn_discrete_scratch_floats(d, n, 0), 4, run_forward, [probs])
    check_exact_size(L.recnn_reinforce_scratch_floats(d, n, chunk), 4, run_grad, [grads, out])


@pytest.mark.parametrize("S,H,I,n,chunk", DISCRETE)
def test_policy_shard_phases(S, H, I, n, chunk):
    """world 1: the stats and gradient phases share one scratch; the forward phase has its own"""
    m, state, action, ret, blp = _discrete(S, H, I, n)
    d, p = m.dims, param_arena(m)
    vs = _lib.VocabShard(0, I, 0, 1)
    rec, frec = (torch.zeros(L.recnn_vocab_record_floats(n), device=DEV) for _ in range(2))
    grads, out, probs = torch.zeros_like(p), torch.zeros(3, device=DEV), torch.zeros(n, I, device=DEV)

    def run_grad(ptr, nbytes):
        st = _lib.stream_ptr()
        return [L.recnn_reinforce_shard_stats(d, vs, p.data_ptr(), state.data_ptr(), action.data_ptr(), n, chunk,
                                              rec.data_ptr(), ptr, st),
                L.recnn_reinforce_shard_grad(d, vs, p.data_ptr(), grads.data_ptr(), state.data_ptr(), action.data_ptr(),
                                             blp.data_ptr(), ret.data_ptr(), n, _lib.REINFORCE_CORRECTED, 1, chunk,
                                             rec.data_ptr(), out.data_ptr(), ptr, st)]

    def run_forward(ptr, nbytes):
        return [L.recnn_discrete_shard_forward(d, vs, p.data_ptr(), state.data_ptr(), n, probs.data_ptr(),
                                               frec.data_ptr(), ptr, _lib.stream_ptr())]
    check_exact_size(L.recnn_reinforce_scratch_floats(d, n, chunk), 4, run_grad, [rec, grads, out])
    check_exact_size(L.recnn_discrete_scratch_floats(d, n, 0), 4, run_forward, [probs, frec])


# ---------------------------------------------------------------- the item-id critic
@pytest.mark.parametrize("S,H,I,n,chunk", DISCRETE)
def test_action_term(S, H, I, n, chunk):
    """the chunked projection from a policy and from dense probabilities, then the critic forward on its result"""
    pp, cp, _, batch, _ = critic_case(S, H, I, n, 5, 1, False)
    policy = make_policy(pp, S, H, I)
    critic = load_net(recnn_b200.nn.Critic(S, I, H), cp, DEV)
    d, pd = _lib.Dims(S, I, H, 0), policy.dims
    state = torch.from_numpy(batch["state"]).to(DEV)
    probs = torch.softmax(torch.randn(n, I, device=DEV), 1)
    term, dense_term, value = (torch.zeros(n, H, device=DEV), torch.zeros(n, H, device=DEV),
                               torch.zeros(n, device=DEV))
    cpar = param_arena(critic).data_ptr()

    def run_policy(ptr, nbytes):
        return [L.recnn_critic_action_term_chunked(
            d, cpar, pd, param_arena(policy).data_ptr(), state.data_ptr(), None, 0, n, chunk, term.data_ptr(), ptr,
            _lib.stream_ptr())]

    def run_dense(ptr, nbytes):
        return [L.recnn_critic_action_term_chunked(
            d, cpar, None, None, None, probs.data_ptr(), I, n, chunk, dense_term.data_ptr(), ptr, _lib.stream_ptr())]

    def run_forward(ptr, nbytes):
        return [L.recnn_critic_forward_action_term(
            d, cpar, state.data_ptr(), term.data_ptr(), n, None, None, value.data_ptr(), ptr, _lib.stream_ptr())]
    check_exact_size(L.recnn_critic_action_term_scratch_floats(d, pd, n, chunk), 4, run_policy, [term])
    check_exact_size(L.recnn_critic_action_term_scratch_floats(d, None, n, chunk), 4, run_dense, [dense_term])
    check_exact_size(L.recnn_forward_scratch_floats(d, n, 0), 4, run_forward, [value])


def _critic_rank(S, H, I, n, chunk, train):
    pp, cp, tcp, batch, masks = critic_case(S, H, I, n, 7, 1, train)
    (rk,), _, _ = critic_ranks(pp, cp, tcp, S, H, I, 1, chunk, batch, masks)       # the rank keeps its batch alive
    a = rk.args
    size = L.recnn_discrete_value_workspace_bytes(a.dims, a.policy_dims, n, a.chunk_items)
    o = rk.opt
    state = [rk.losses, rk.rng_step, param_arena(rk.value), grad_arena(rk.value)]
    state += [t for t in (o._m, o._v, o._t, o._slow) if t is not None]
    return rk, size, state


@pytest.mark.parametrize("S,H,I,n,chunk", DISCRETE)
def test_item_id_critic_step(S, H, I, n, chunk):
    rk, size, state = _critic_rank(S, H, I, n, chunk, train=chunk == 128)

    def run(ptr, nbytes):
        rk.args.workspace, rk.args.workspace_bytes = ptr, nbytes
        return [L.recnn_discrete_value_step(rk.args, _lib.stream_ptr())]
    check_exact_size(size, 1, run, state)
    check_too_small(size, run)


@pytest.mark.parametrize("S,H,I,n,chunk", DISCRETE)
def test_item_id_critic_shard_phases(S, H, I, n, chunk):
    """world 1: begin, merge and end on one workspace (the all-gather and the all-reduce are the identity)"""
    rk, size, state = _critic_rank(S, H, I, n, chunk, train=chunk != 128)
    rec, terms = torch.zeros(L.recnn_vocab_record_floats(n), device=DEV), torch.zeros(2 * n * H, device=DEV)

    def run(ptr, nbytes):
        st = _lib.stream_ptr()
        rk.args.workspace, rk.args.workspace_bytes = ptr, nbytes
        return [L.recnn_discrete_value_shard_begin(rk.args, rk.shard, rec.data_ptr(), st),
                L.recnn_discrete_value_shard_merge(rk.args, rk.shard, rec.data_ptr(), terms.data_ptr(), st),
                L.recnn_discrete_value_shard_end(rk.args, rk.shard, terms.data_ptr(), st)]
    check_exact_size(size, 1, run, state + [rec, terms])
    check_too_small(size, run)


# ---------------------------------------------------------------- the behaviour policy beta
@pytest.mark.parametrize("S,H,I,n,chunk", DISCRETE)
def test_beta_step(S, H, I, n, chunk):
    torch.manual_seed(S + I)
    beta = recnn_b200.nn.Beta(S, I).to(DEV)
    o = beta.optim
    state_in = torch.randn(n, S, device=DEV)
    action = torch.randint(0, I, (n,), device=DEV)
    probs, loss = torch.zeros(n, I, device=DEV), torch.zeros((), device=DEV)
    error = torch.zeros(1, dtype=torch.int32, device=DEV)
    a = _lib.BetaArgs()
    a.dims, a.n_rows, a.chunk_items = beta.dims, n, chunk
    a.net, a.optim = o.c_net(beta), o.c_optim()
    a.state, a.state_ld, a.action = state_in.data_ptr(), S, action.data_ptr()
    a.probs_out, a.loss, a.error = probs.data_ptr(), loss.data_ptr(), error.data_ptr()
    state = [probs, loss, error, param_arena(beta), grad_arena(beta)]
    state += [t for t in (o._m, o._v, o._t, o._slow) if t is not None]

    def run(ptr, nbytes):
        a.workspace, a.workspace_bytes = ptr, nbytes
        return [L.recnn_beta_step(a, _lib.stream_ptr())]
    size = L.recnn_beta_workspace_bytes(beta.dims, n, chunk)
    check_exact_size(size, 1, run, state)
    check_too_small(size, run)


# ---------------------------------------------------------------- retrieval
@pytest.mark.parametrize("nq,items,dim,k,metric", [(5, 1000, 32, 10, _lib.METRIC_L2),      # tensor-core scores
                                                   (7, 3001, 13, 20, _lib.METRIC_COS)])    # CUDA-core scores
def test_retrieval(nq, items, dim, k, metric):
    torch.manual_seed(items)
    table, queries = torch.randn(items, dim, device=DEV), torch.randn(nq, dim, device=DEV)
    norms = torch.empty(items, device=DEV)
    _lib.check(L.recnn_item_norms(table.data_ptr(), items, dim, metric, norms.data_ptr(), _lib.stream_ptr()))
    ids, dist = torch.zeros(nq, k, dtype=torch.int64, device=DEV), torch.zeros(nq, k, device=DEV)

    def run(ptr, nbytes):
        return [L.recnn_retrieve_topk(queries.data_ptr(), nq, dim, table.data_ptr(), items, norms.data_ptr(), metric,
                                      k, ids.data_ptr(), dist.data_ptr(), ptr, nbytes, _lib.stream_ptr())]
    size = L.recnn_retrieve_workspace_bytes(nq, items, k)
    check_exact_size(size, 1, run, [ids, dist])
    check_too_small(size, run)
