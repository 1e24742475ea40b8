"""REINFORCE policy gradient over item chunks (recnn_reinforce_policy_grad_chunked) on the GPU: against the float64
oracle, against the single-chunk call on identical inputs, bit-for-bit determinism, a 262,144-item vocabulary through
the public API (automatic chunking, bounded memory), an agent loop that chunks, and the error paths."""
from __future__ import annotations

import ctypes
import gc

import numpy as np
import pytest
import torch

import recnn_b200
from recnn_b200 import _lib
from recnn_b200.nn.arena import param_arena, grad_arena
from recnn_b200.nn.update import reinforce as RF
from oracle import reinforce_oracle as RO
from tests._discrete import make_policy

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
METHODS = ["basic_reinforce", "reinforce_with_correction", "reinforce_with_TopK_correction"]
# chunked vs single chunk: both are fp32 with 3xTF32 contractions; only the order of the softmax sum (merged per
# chunk), the split-K order of dW2 (per chunk width) and of dh (accumulated chunk by chunk) differ
REORDER_BAR = 1e-5


def unpack(g, m):
    """{w1, b1, w2, b2} views of a flat gradient arena of policy m."""
    d = m.dims
    buf = (ctypes.c_int64 * 7)()
    _lib.check(_lib.lib().recnn_discrete_layout(d, buf))
    w1, b1, w2, b2, ld1, ld2, _ = list(buf)
    S, H, I = d.state_dim, d.hidden, d.num_items
    return {"w1": g[w1:w1 + H * ld1].view(H, ld1)[:, :S], "b1": g[b1:b1 + H],
            "w2": g[w2:w2 + I * ld2].view(I, ld2)[:, :H], "b2": g[b2:b2 + I]}


def policy_grad(m, state, action, blp, ret, method, K, chunk):
    """(loss, oob flag, gradient dict) of one explicit recnn_reinforce_policy_grad_chunked call."""
    L = _lib.lib()
    d = m.dims
    n = state.shape[0]
    flat = param_arena(m)
    grads = torch.full_like(flat, float("nan"))           # every gradient entry must be written
    scratch = torch.empty(L.recnn_reinforce_scratch_floats(d, n, chunk), device=DEV)
    out = torch.zeros(2, device=DEV)
    _lib.check(L.recnn_reinforce_policy_grad_chunked(d, flat.data_ptr(), grads.data_ptr(), state.data_ptr(),
                                                     action.data_ptr(), _lib.ptr(blp), ret.data_ptr(), n, method, K,
                                                     chunk, out.data_ptr(), scratch.data_ptr(), _lib.stream_ptr()))
    torch.cuda.synchronize()
    return float(out[0]), int(out.view(torch.int32)[1]), unpack(grads, m)


def edge_actions(rng, n, I, chunk):
    """random actions, with the first and last column of a chunk, the first column of the last chunk and the last item"""
    a = rng.integers(0, I, n)
    last0 = (I - 1) // chunk * chunk
    edges = [0, chunk - 1, min(chunk, I - 1), last0, I - 1, I - 1 - (I - last0) // 2]
    a[:len(edges)] = edges
    return a


def case(S, H, I, R, seed):
    rng = np.random.default_rng(seed)
    p = RO.make_discrete_actor(rng, S, I, H)
    state = rng.normal(0, 1, (R, S)).astype(np.float32)
    blp = np.log(rng.uniform(1e-4, 5e-4, R)).astype(np.float32)
    ret = rng.normal(0, 1, R).astype(np.float32)
    return rng, p, state, blp, ret


def rel_diff(a, b):
    return float((a - b).abs().max() / b.abs().max())


SHAPES = [(52, 64, 1000, 40, 128),        # last chunk 104 wide (tensor cores)
          (52, 64, 1003, 40, 128),        # last chunk 107 wide (exact-fp32 SIMT path)
          (1290, 256, 5000, 320, 512)]


@pytest.mark.parametrize("method", METHODS)
@pytest.mark.parametrize("S,H,I,R,chunk", SHAPES)
@pytest.mark.parametrize("single", [False, True], ids=["chunked", "single"])
def test_chunked_matches_oracle(method, S, H, I, R, chunk, single):
    rng, p, state, blp, ret = case(S, H, I, R, S + I + R)
    if single:
        chunk_used = I
    else:
        chunk_used = chunk
    action = edge_actions(rng, R, I, chunk)
    mid = RO.METHODS[method]
    m = make_policy(p, S, H, I)
    loss, oob, got = policy_grad(m, torch.from_numpy(state).to(DEV), torch.from_numpy(action).to(DEV),
                                 None if mid == RO.BASIC else torch.from_numpy(blp).to(DEV),
                                 torch.from_numpy(ret).to(DEV), mid, 10, chunk_used)
    want_loss, want, _ = RO.reinforce_policy_grad(p, state, action, None if mid == RO.BASIC else blp, ret, mid, 10)
    assert oob == 0
    assert loss == pytest.approx(want_loss, rel=2e-4, abs=1e-4 * (1 + abs(want_loss)))
    for k in ("w1", "b1", "w2", "b2"):
        scale = np.abs(want[k]).max()
        assert scale > 0
        err = np.abs(got[k].cpu().numpy() - want[k]).max()
        assert err <= 3e-4 * scale, (k, err, scale)


@pytest.mark.parametrize("S,H,I,R,chunk", SHAPES)
def test_chunked_matches_single_chunk_and_is_deterministic(S, H, I, R, chunk):
    rng, p, state, blp, ret = case(S, H, I, R, 7 * S + I)
    action = torch.from_numpy(edge_actions(rng, R, I, chunk)).to(DEV)
    m = make_policy(p, S, H, I)
    args = (torch.from_numpy(state).to(DEV), action, torch.from_numpy(blp).to(DEV), torch.from_numpy(ret).to(DEV),
            RO.TOPK, 10)
    l1, _, single = policy_grad(m, *args, I)
    l2, _, chunked = policy_grad(m, *args, chunk)
    l3, _, again = policy_grad(m, *args, chunk)
    assert l2 == pytest.approx(l1, rel=1e-5, abs=1e-6)
    assert l3 == l2
    for k in single:
        assert torch.isfinite(chunked[k]).all(), k
        assert torch.equal(chunked[k], again[k]), k
        r = rel_diff(chunked[k], single[k])
        print("%s chunk %d %s: max |chunked - single| / max |single| = %.2e" % ((S, H, I, R), chunk, k, r))
        assert r <= REORDER_BAR, (k, r)


def _torch_reference(m, state, action, blp, ret, method, K, block=512):
    """float64 loss and gradients on the GPU, in row blocks of the [R, num_items] probabilities."""
    f = {k: v.detach().double() for k, v in (("w1", m.linear1.weight), ("b1", m.linear1.bias),
                                              ("w2", m.linear2.weight), ("b2", m.linear2.bias))}
    g = {k: torch.zeros_like(v) for k, v in f.items()}
    loss = abs_sum = 0.0
    for r0 in range(0, state.shape[0], block):
        s = state[r0:r0 + block].double()
        a = action[r0:r0 + block]
        h = torch.relu(s @ f["w1"].T + f["b1"])
        probs = torch.softmax(h @ f["w2"].T + f["b2"], dim=1)
        pa = probs.gather(1, a[:, None])[:, 0]
        L, gr, _ = RO.row_terms(pa.cpu().numpy(), None if blp is None else blp[r0:r0 + block].cpu().numpy(),
                                ret[r0:r0 + block].cpu().numpy(), method, K)
        loss += float(L.sum())
        abs_sum += float(np.abs(L).sum())
        gr = torch.from_numpy(gr).to(DEV)
        dz = -probs * gr[:, None]
        dz[torch.arange(dz.shape[0], device=DEV), a] += gr
        g["w2"] += dz.T @ h
        g["b2"] += dz.sum(0)
        dh = (dz @ f["w2"]) * (h > 0)
        g["w1"] += dh.T @ s
        g["b1"] += dh.sum(0)
        del probs, dz
    return loss, abs_sum, g


def _choose_reinforce_returns(rewards):
    """ChooseREINFORCE.__call__'s normalised discounted returns, with the same torch float32 arithmetic"""
    R, out = 0, []
    for r in [torch.tensor(x) for x in rewards][::-1]:
        R = r + 0.99 * R
        out.insert(0, R)
    out = torch.tensor(out)
    return (out - out.mean()) / (out.std() + 0.0001)


def test_large_vocabulary_through_the_public_api(monkeypatch):
    """262,144 items x 4,096 saved rows: the [rows, items] logits (4.3 GB) exceed the budget, so ChooseREINFORCE chunks
    by itself; gradients match the single-chunk call and a float64 reference, and the call's extra memory stays near
    one logits chunk."""
    S, H, I, N, T = 1290, 256, 262_144, 1024, 4
    R = N * T
    torch.manual_seed(17)
    with torch.device(DEV):
        m = recnn_b200.nn.DiscreteActor(S, I, H)
    gen = torch.Generator(device=DEV).manual_seed(3)
    states = torch.randn(T, N, S, device=DEV, generator=gen)
    actions = torch.randint(0, I, (T, N), device=DEV, generator=gen)
    actions[0, :3] = torch.tensor([0, I - 1, RF._chunk_items(R, I)], device=DEV)
    blp = torch.log(torch.empty(T, N, device=DEV).uniform_(1e-6, 5e-6, generator=gen))
    rewards = [float(x) for x in np.random.default_rng(4).normal(0, 1, T)]
    for t in range(T):
        m._saved.append({"state": states[t], "action": actions[t], "beta_log_prob": blp[t], "K": 10})
        m.rewards.append(torch.tensor(rewards[t], device=DEV))
    grad_arena(m)                                                   # allocated before the measured call
    chosen = []
    pick = RF._chunk_items
    monkeypatch.setattr(RF, "_chunk_items", lambda n, items: chosen.append(pick(n, items)) or chosen[-1])
    gc.collect()                                                    # earlier tests' modules (reference cycles)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.max_memory_allocated()
    loss =recnn_b200.nn.ChooseREINFORCE(recnn_b200.nn.ChooseREINFORCE.reinforce_with_TopK_correction)(m, None, learn=False)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    assert chosen and chosen[0] < I and chosen[0] % 128 == 0
    chunk = chosen[0]
    scratch = _lib.lib().recnn_reinforce_scratch_floats(m.dims, R, chunk) * 4
    single = _lib.lib().recnn_reinforce_scratch_floats(m.dims, R, I) * 4
    bound = RF._LOGITS_BUDGET_BYTES + R * ((S + 3) // 4 * 4 + 2 * H) * 4 + 2 * (chunk + 65536) * (H + 1) * 4
    print("chunk %d: peak extra %.3f GB, scratch %.3f GB, single-chunk scratch %.3f GB"
          % (chunk, peak / 1e9, scratch / 1e9, single / 1e9))
    assert scratch <= bound
    assert peak <= bound + R * S * 4 + (64 << 20)                    # + the concatenated saved states, small slack
    assert peak < single / 2
    got = {k: v.clone() for k, v in unpack(grad_arena(m), m).items()}

    state, action, beta = states.reshape(R, S), actions.reshape(R), blp.reshape(R)
    ret = _choose_reinforce_returns(rewards).to(DEV).repeat_interleave(N)
    l64, abs_sum, want = _torch_reference(m, state, action, beta, ret, RO.TOPK, 10)
    l1, _, want1 = policy_grad(m, state, action, beta, ret, RO.TOPK, 10, I)
    # the loss is a sum of signed row terms that largely cancel: reordering is measured against the sum of |terms|
    print("262144 items, chunk %d vs single, loss: %.2e of sum |row terms|" % (chunk, abs(float(loss) - l1) / abs_sum))
    assert abs(float(loss) - l1) <= 1e-6 * abs_sum
    for k in got:
        r = rel_diff(got[k], want1[k])
        print("262144 items, chunk %d vs single, %s: %.2e" % (chunk, k, r))
        assert r <= REORDER_BAR, (k, r)
    del want1
    assert float(loss) == pytest.approx(l64, rel=2e-4, abs=1e-4 * (1 + abs(l64)))
    for k in got:
        scale = float(want[k].abs().max())
        err = float((got[k].double() - want[k]).abs().max())
        assert err <= 3e-4 * scale, (k, err, scale)


def _agent_run(budget, monkeypatch, S=52, H=64, I=301, N=10, steps=21):
    monkeypatch.setattr(RF, "_LOGITS_BUDGET_BYTES", budget)
    torch.manual_seed(5)
    rng = np.random.default_rng(8)
    policy = recnn_b200.nn.DiscreteActor(S, I, H)
    value = recnn_b200.nn.Critic(S, I, H, 54e-2)
    agent = recnn_b200.nn.Reinforce(policy, value).to(torch.device(DEV))
    policy = agent.nets["policy_net"]
    bw = torch.from_numpy(rng.normal(0, 0.3, (I, S)).astype(np.float32)).to(DEV)

    def select_action_corr(state, action, K, writer, step, **kwargs):
        beta = lambda s, action=None: torch.softmax(s @ bw.T, dim=1)       # noqa: E731
        return agent.nets["policy_net"]._select_action_with_TopK_correction(state, beta, action, K=K, writer=writer, step=step)

    policy.select_action = select_action_corr
    agent.params["reinforce"] = recnn_b200.nn.ChooseREINFORCE(recnn_b200.nn.ChooseREINFORCE.reinforce_with_TopK_correction)
    agent.params["K"] = 10
    agent.optimizers["policy_optimizer"] = torch.optim.SGD(policy.parameters(), lr=1e-2)
    agent.optimizers["value_optimizer"] = recnn_b200.optim.Adam(agent.nets["value_net"].parameters(), lr=1e-3)
    out = []
    for _ in range(steps):
        one_hot = np.zeros((N, I), np.float32)
        one_hot[np.arange(N), rng.integers(0, I, N)] = 1
        b = {"state": rng.normal(0, 1, (N, S)).astype(np.float32), "action": one_hot,
             "reward": rng.integers(1, 6, N).astype(np.float32) - 3,
             "next_state": rng.normal(0, 1, (N, S)).astype(np.float32), "done": (rng.random(N) < 0.1).astype(np.float32)}
        out.append(agent.update({k: torch.from_numpy(v) for k, v in b.items()}))
        agent.step()
    return out, {k: v.detach().clone() for k, v in policy.named_parameters()}


def test_agent_loop_with_chunked_policy_steps(monkeypatch):
    """Reinforce.update with a budget small enough that every policy step chunks (100 rows x 301 items -> chunks of
    128, 128, 45; the last one on the SIMT path): the same losses and stepped weights as the single-chunk run."""
    want_out, want_w = _agent_run(1 << 30, monkeypatch)
    assert RF._chunk_items(100, 301) == 301
    got_out, got_w = _agent_run(100 * 128 * 4, monkeypatch)
    assert RF._chunk_items(100, 301) == 128
    assert [o is not None for o in got_out] == [o is not None for o in want_out] == [i in (10, 20) for i in range(21)]
    for g, w in zip(got_out, want_out):
        if w is None:
            continue
        assert g["value"] == pytest.approx(w["value"], rel=2e-4, abs=1e-6)
        assert g["policy"] == pytest.approx(w["policy"], rel=2e-4, abs=1e-4 * (1 + abs(w["policy"])))
    for k in want_w:
        scale = float(want_w[k].abs().max())
        err = float((got_w[k] - want_w[k]).abs().max())
        assert err <= 1e-5 * scale, (k, err, scale)


def test_errors(monkeypatch):
    rng, p, state, blp, ret = case(52, 64, 1000, 40, 1)
    m = make_policy(p, 52, 64, 1000)
    args = (torch.from_numpy(state).to(DEV), torch.from_numpy(rng.integers(0, 1000, 40)).to(DEV), None,
            torch.from_numpy(ret).to(DEV), RO.BASIC, 1)
    for bad in (100, 129, 0, -128, 1024, 1001):
        flat = param_arena(m)
        out = torch.zeros(2, device=DEV)
        scratch = torch.empty(1 << 20, device=DEV)
        with pytest.raises(_lib.RecnnError):
            _lib.check(_lib.lib().recnn_reinforce_policy_grad_chunked(
                m.dims, flat.data_ptr(), torch.zeros_like(flat).data_ptr(), args[0].data_ptr(), args[1].data_ptr(),
                None, args[3].data_ptr(), 40, RO.BASIC, 1, bad, out.data_ptr(), scratch.data_ptr(), _lib.stream_ptr()))
    # an action id == num_items on a chunked policy step
    monkeypatch.setattr(RF, "_LOGITS_BUDGET_BYTES", 4 * 256 * 4)
    assert RF._chunk_items(4, 1000) == 256
    m._saved.append({"state": args[0][:2], "action": torch.tensor([1, 1000], device=DEV), "beta_log_prob": None})
    m._saved.append({"state": args[0][2:4], "action": torch.tensor([999, 0], device=DEV), "beta_log_prob": None})
    m.rewards += [torch.tensor(1.0), torch.tensor(2.0)]
    with pytest.raises(IndexError):
        recnn_b200.nn.ChooseREINFORCE()(m, torch.optim.SGD(m.parameters(), lr=0.1))
