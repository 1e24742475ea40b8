"""REINFORCE critic with item-id actions (recnn_discrete_value_step, recnn_critic_action_term_chunked) on the GPU:
parity with the float64 oracle fed the equivalent one-hot and with the dense CUDA path, the structure and determinism
of the action block's gradient, the chunked projection against float64, a million items on one GPU with bounded
memory, an agent loop over item-id batches, and the error paths."""
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
from recnn_b200.nn.arena import grad_arena
from recnn_b200.nn.update import _ids
from recnn_b200.nn.update import reinforce as RF
from oracle import recnn_oracle as O
from oracle import reinforce_oracle as RO
from tests._cuda import load_net, dump_net

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def make_policy(p, S, H, I):
    m = recnn_b200.nn.DiscreteActor(S, I, H)
    with torch.no_grad():
        for lin, w, b in ((m.linear1, "w1", "b1"), (m.linear2, "w2", "b2")):
            lin.weight.copy_(torch.from_numpy(p[w]))
            lin.bias.copy_(torch.from_numpy(p[b]))
    return m.to(DEV)


def make_agent(pp, cp, S, H, I, train):
    policy = make_policy(pp, S, H, I)
    value = load_net(recnn_b200.nn.Critic(S, I, H, 0.3), cp, DEV)
    algo = recnn_b200.nn.Reinforce(policy, value)
    algo.nets["value_net"].train(train)
    algo.optimizers["value_optimizer"] = recnn_b200.optim.Adam(algo.nets["value_net"].parameters(), lr=1e-3)
    return algo


def ids_batch(rng, N, S, I, edges=()):
    action = rng.integers(0, I, N)
    k = N // 4
    action[:k] = action[k:2 * k]                                 # repeated ids across rows
    for i, e in enumerate(edges):
        action[N // 2 + i] = e
    return {"state": rng.normal(0, 1, (N, S)).astype(np.float32), "action": action.astype(np.int64),
            "reward": rng.integers(1, 6, N).astype(np.float32) - 3, "next_state": rng.normal(0, 1, (N, S)).astype(np.float32),
            "done": (rng.random(N) < 0.1).astype(np.float32)}


def one_hot(b, I):
    d = dict(b)
    oh = np.zeros((len(b["action"]), I), np.float32)
    oh[np.arange(len(b["action"])), b["action"]] = 1
    d["action"] = oh
    return d


def to_dev(b):
    return {k: (torch.from_numpy(v) if isinstance(v, np.ndarray) else v) for k, v in b.items()}


CASES = [(52, 64, 300, 24, None), (1290, 256, 5000, 256, 1280)]      # chunk 1280: four chunks, the last 1160 wide


@pytest.mark.parametrize("train", [False, True], ids=["eval", "train"])
@pytest.mark.parametrize("S,H,I,N,chunk", CASES, ids=["small", "notebook"])
def test_ids_match_oracle_and_dense_path(S, H, I, N, chunk, train, monkeypatch):
    """Three Adam steps through value_update with item ids against the oracle fed the one-hot (loss rel 2e-5, weights
    rtol 1e-4 / atol 1e-5 of the largest) and against the dense CUDA path on the same inputs."""
    if chunk is not None:
        monkeypatch.setattr(RF, "_chunk_items", lambda n, items: chunk)
    rng = np.random.default_rng(S + N + int(train))
    pp = RO.make_discrete_actor(rng, S, I, H)
    cp = O.make_critic(rng, S, I, H, 0.3)
    ids_algo, dense_algo = make_agent(pp, cp, S, H, I, train), make_agent(pp, cp, S, H, I, train)
    o_nets = {"value_net": O.copy_net(cp), "target_value_net": O.copy_net(cp), "target_policy_net": pp}
    o_opts = {"value_optimizer": O.make_optimizer("adam", lr=1e-3)}
    params = dict(ids_algo.params)
    edges = (0, I - 1) + ((chunk, chunk - 1, 2 * chunk) if chunk else ())
    for step in range(3):
        b = ids_batch(rng, N, S, I, edges)
        masks = None
        if train:
            masks = [(rng.random((N, H)) >= 0.5).astype(np.uint8) for _ in range(2)]
        want, _ = RO.value_update(one_hot(b, I), params, o_nets, o_opts, masks, learn=True)
        extra = {} if masks is None else {"dropout_masks": [torch.from_numpy(m) for m in masks * 3]}
        got = recnn_b200.nn.value_update({**to_dev(b), **extra}, params, ids_algo.nets, ids_algo.optimizers,
                                         torch.device(DEV), {}, learn=True, step=step)
        dense = recnn_b200.nn.value_update({**to_dev(one_hot(b, I)), **extra}, params, dense_algo.nets,
                                           dense_algo.optimizers, torch.device(DEV), {}, learn=True, step=step)
        assert float(got) == pytest.approx(float(want), rel=2e-5, abs=1e-6)
        assert float(got) == pytest.approx(float(dense), rel=1e-5, abs=1e-7)
    after, after_dense = dump_net(ids_algo.nets["value_net"]), dump_net(dense_algo.nets["value_net"])
    for t in O.PARAM_ORDER:
        w = o_nets["value_net"][t]
        bar = 1e-4 * np.abs(w) + 1e-5 * np.abs(w).max()
        if chunk is None:
            np.testing.assert_allclose(after[t], w, rtol=1e-4, atol=1e-5 * np.abs(w).max(), err_msg=t)
            assert np.abs(after[t] - after_dense[t]).max() <= 2e-6 * np.abs(w).max(), t
        else:
            # Adam's step g / (|g| + eps) turns the fp32 rounding of a gradient that nearly cancels into an lr-sized
            # difference.  Among the 1.6M layer-1 weights of this shape a handful of such elements exist, and the dense
            # CUDA path misses the bar on them just as the item-id path does (up to 14 layer-1 weights on these seeds, either path):
            # everything else must hold the bar, and the outliers stay a handful per tensor.
            out_ids = int((np.abs(after[t] - w) > bar).sum())
            out_dense = int((np.abs(after_dense[t] - w) > bar).sum())
            out_pair = int((np.abs(after[t] - after_dense[t]) > bar).sum())
            print("%s %s: outside the oracle bar: item ids %d, dense %d; ids vs dense %d of %d"
                  % (t, "train" if train else "eval", out_ids, out_dense, out_pair, w.size))
            assert max(out_ids, out_pair) <= 16, t


def _float64_critic_grads(algo, b, S, I, params):
    """float64 autograd of misc.py:28-41 with the one-hot action: loss and d loss / d linear1.weight"""
    f = lambda t: t.detach().double()                                  # noqa: E731
    v, tv, tp = algo.nets["value_net"], algo.nets["target_value_net"], algo.nets["target_policy_net"]
    s, s2 = (torch.from_numpy(b[k]).to(DEV).double() for k in ("state", "next_state"))
    r, d = (torch.from_numpy(b[k]).to(DEV).double()[:, None] for k in ("reward", "done"))
    a = torch.zeros(len(b["action"]), I, device=DEV, dtype=torch.float64)
    a[torch.arange(len(b["action"])), torch.from_numpy(b["action"]).to(DEV)] = 1
    probs = torch.softmax(torch.relu(s2 @ f(tp.linear1.weight).T + f(tp.linear1.bias)) @ f(tp.linear2.weight).T
                          + f(tp.linear2.bias), 1)

    def critic(net, x, act, w1=None):
        h = torch.relu(torch.cat([x, act], 1) @ (f(net.linear1.weight) if w1 is None else w1).T + f(net.linear1.bias))
        h = torch.relu(h @ f(net.linear2.weight).T + f(net.linear2.bias))
        return h @ f(net.linear3.weight).T + f(net.linear3.bias)

    y = (r + (1 - d) * params["gamma"] * critic(tv, s2, probs)).clamp(params["min_value"], params["max_value"])
    w1 = f(v.linear1.weight).requires_grad_(True)
    loss = ((critic(v, s, a, w1) - y) ** 2).mean()
    loss.backward()
    return float(loss), w1.grad


def test_action_block_gradient_structure_and_determinism(monkeypatch):
    """External optimizer (SGD, lr 0): .grad of linear1.weight read back.  Unselected action columns are exactly 0, the
    selected ones match float64 segmented sums, and two identical calls give identical bits."""
    S, H, I, N = 1290, 256, 5000, 256
    monkeypatch.setattr(RF, "_chunk_items", lambda n, items: 1280)
    rng = np.random.default_rng(5)
    algo = make_agent(RO.make_discrete_actor(rng, S, I, H), O.make_critic(rng, S, I, H, 0.3), S, H, I, False)
    algo.optimizers["value_optimizer"] = torch.optim.SGD(algo.nets["value_net"].parameters(), lr=0.0)
    b = ids_batch(rng, N, S, I, (0, I - 1, 1280, 1279))
    params = dict(algo.params)
    runs = []
    for _ in range(2):
        loss = recnn_b200.nn.value_update(to_dev(b), params, algo.nets, algo.optimizers, torch.device(DEV), {},
                                          learn=True)
        runs.append((float(loss), [p.grad.clone() for p in algo.nets["value_net"].parameters()]))
    assert runs[0][0] == runs[1][0]
    for g0, g1 in zip(runs[0][1], runs[1][1]):
        assert torch.equal(g0, g1)
    gw1 = runs[0][1][0]
    block = gw1[:, S:]
    hit = np.zeros(I, bool)
    hit[b["action"]] = True
    assert int((block[:, torch.from_numpy(~hit).to(DEV)] != 0).sum()) == 0         # exactly 0.0 where no row selected
    l64, g64 = _float64_critic_grads(algo, b, S, I, params)
    assert runs[0][0] == pytest.approx(l64, rel=2e-5)
    want = g64[:, S:]
    scale = float(want.abs().max())
    assert float((block.double() - want).abs().max()) <= 1e-4 * scale
    assert float((gw1[:, :S].double() - g64[:, :S]).abs().max()) <= 1e-4 * float(g64[:, :S].abs().max())


def _projection_case(S, H, Hp, I, N, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    with torch.device(DEV):
        policy = recnn_b200.nn.DiscreteActor(S, I, Hp)
        value = recnn_b200.nn.Critic(S, I, H)
    state = torch.randn(N, S, device=DEV, generator=g)
    w = lambda t: t.detach().double()                                  # noqa: E731
    logits = torch.relu(state.double() @ w(policy.linear1.weight).T + w(policy.linear1.bias)) @ w(policy.linear2.weight).T
    probs = torch.softmax(logits + w(policy.linear2.bias), 1)
    want = probs @ w(value.linear1.weight)[:, S:].T
    return policy, value, state, probs, want


def _check_projection(S, H, Hp, I, N, widths):
    policy, value, state, probs, want = _projection_case(S, H, Hp, I, N, S + I)
    scale = float(want.abs().max())
    for chunk in widths:
        for src in ("policy", "dense"):
            if src == "policy":
                got = _ids.critic_action_term(value, policy=policy, state=state, chunk_items=chunk)
            else:
                got = _ids.critic_action_term(value, probs=probs.float(), chunk_items=chunk)
            err = float((got.double() - want).abs().max())
            print("projection S=%d I=%d chunk=%d %s: %.2e of max" % (S, I, chunk, src, err / scale))
            assert err <= 1e-5 * scale, (chunk, src, err, scale)


@pytest.mark.parametrize("S,H,Hp,I,N", [(1290, 256, 256, 5000, 96), (52, 64, 32, 300, 24), (2570, 256, 256, 4096, 40)])
def test_projection_matches_float64(S, H, Hp, I, N):
    _check_projection(S, H, Hp, I, N, [I, 128, 1280 if I > 1280 else 256])


def test_projection_on_the_cuda_core_back_end():
    """The same check with every GEMM on the exact-fp32 CUDA-core kernel (the back end taken where the tensor cores'
    TMA cannot address an operand), in a process of its own (the back end is fixed per process)."""
    code = ("import sys; sys.path.insert(0, %r); from tests import test_reinforce_critic_ids_gpu as T; "
            "T._check_projection(1290, 256, 256, 3000, 40, [3000, 128, 1024]); "
            "T._check_projection(52, 64, 32, 300, 24, [300, 128])" % ROOT)
    env = dict(os.environ, RECNN_B200_MATH="simt")
    r = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, cwd=ROOT)
    print(r.stdout[-2000:], r.stderr[-2000:])
    assert r.returncode == 0


def _million_item_nets(S, H, I):
    torch.manual_seed(23)
    with torch.device(DEV):
        policy = recnn_b200.nn.DiscreteActor(S, I, H)
        value = recnn_b200.nn.Critic(S, I, H, 3e-3)
    algo = recnn_b200.nn.Reinforce(policy, value)
    algo.nets["value_net"].eval()
    return algo


def _big_batch(N, S, I, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    action = torch.randint(0, I, (N,), device=DEV, generator=g)
    action[:4] = torch.tensor([0, I - 1, 5, 5], device=DEV)
    return {"state": torch.randn(N, S, device=DEV, generator=g), "next_state": torch.randn(N, S, device=DEV, generator=g),
            "action": action, "reward": torch.randint(1, 6, (N,), device=DEV, generator=g).float() - 3,
            "done": (torch.rand(N, device=DEV, generator=g) < 0.1).float()}


def _chunked_float64_loss(algo, b, params, rows=256):
    f = lambda t: t.detach().double()                                  # noqa: E731
    v, tv, tp = algo.nets["value_net"], algo.nets["target_value_net"], algo.nets["target_policy_net"]
    S = v.linear1.in_features - tp.linear2.out_features
    total = 0.0
    for r0 in range(0, b["state"].shape[0], rows):
        sl = slice(r0, r0 + rows)
        s, s2, a = b["state"][sl].double(), b["next_state"][sl].double(), b["action"][sl]
        probs = torch.softmax(torch.relu(s2 @ f(tp.linear1.weight).T + f(tp.linear1.bias)) @ f(tp.linear2.weight).T
                              + f(tp.linear2.bias), 1)
        ht = torch.relu(s2 @ f(tv.linear1.weight)[:, :S].T + probs @ f(tv.linear1.weight)[:, S:].T + f(tv.linear1.bias))
        del probs
        qt = torch.relu(ht @ f(tv.linear2.weight).T + f(tv.linear2.bias)) @ f(tv.linear3.weight).T + f(tv.linear3.bias)
        y = (b["reward"][sl].double()[:, None] + (1 - b["done"][sl].double()[:, None]) * params["gamma"] * qt)
        y = y.clamp(params["min_value"], params["max_value"])
        h = torch.relu(s @ f(v.linear1.weight)[:, :S].T + f(v.linear1.weight)[:, S + a].T + f(v.linear1.bias))
        q = torch.relu(h @ f(v.linear2.weight).T + f(v.linear2.bias)) @ f(v.linear3.weight).T + f(v.linear3.bias)
        total += float(((q - y) ** 2).sum())
    return total / b["state"].shape[0]


def _measured_call(algo, b, params):
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.max_memory_allocated()
    loss = recnn_b200.nn.value_update(b, params, algo.nets, algo.optimizers, torch.device(DEV), {}, learn=True)
    torch.cuda.synchronize()
    return float(loss), torch.cuda.max_memory_allocated() - base


def _memory_bound(algo, N, S, H, I):
    chunk = RF._chunk_items(N, I)
    d, pd = _ids._critic_dims(algo.nets["value_net"], I), algo.nets["target_policy_net"].dims
    ws = _lib.lib().recnn_discrete_value_workspace_bytes(d, pd, N, chunk)
    # the workspace (one [N, chunk] logits chunk + [N, H] buffers) and the staged batch, plus a little allocator slack
    return ws, ws + N * (2 * S + 4) * 4 + (64 << 20)


@pytest.mark.parametrize("N", [2048, 16384])
def test_million_items_on_one_gpu(N):
    """S 2570 / H 256 / 1,048,576 items.  At 2,048 rows the loss matches a chunked float64 reference; at 16,384 rows the
    call completes, finite and deterministic.  Peak extra memory stays within the chunk-sized workspace, far below one
    [N, num_items] fp32 matrix."""
    S, H, I = 2570, 256, 1 << 20
    algo = _million_item_nets(S, H, I)
    params = dict(algo.params)
    warm = _big_batch(8, S, I, 1)
    recnn_b200.nn.value_update(warm, params, algo.nets, algo.optimizers, torch.device(DEV), {}, learn=True)   # arenas
    b = _big_batch(N, S, I, 2)
    ws, bound = _memory_bound(algo, N, S, H, I)
    if N == 2048:
        want = _chunked_float64_loss(algo, b, params)
    v0 = algo.nets["value_net"].linear1.weight.detach()[:, S + 5].clone()
    loss, peak = _measured_call(algo, b, params)
    print("N=%d: loss %.6g, peak extra %.3f GB, workspace %.3f GB, one [N, items] matrix %.1f GB"
          % (N, loss, peak / 1e9, ws / 1e9, N * I * 4 / 1e9))
    assert np.isfinite(loss)
    assert peak <= bound and peak < N * I * 4 / 4
    assert not torch.equal(v0, algo.nets["value_net"].linear1.weight.detach()[:, S + 5])
    if N == 2048:
        assert loss == pytest.approx(want, rel=2e-4)
    else:
        # determinism: the same call from the same weights (SGD at lr 0 leaves them in place) gives identical bits
        algo.optimizers["value_optimizer"] = torch.optim.SGD(algo.nets["value_net"].parameters(), lr=0.0)
        runs = []
        for _ in range(2):
            l = recnn_b200.nn.value_update(b, params, algo.nets, algo.optimizers, torch.device(DEV), {}, learn=True)
            runs.append((float(l), algo.nets["value_net"].linear1.weight.grad.clone()))
        assert runs[0][0] == runs[1][0] and torch.equal(runs[0][1], runs[1][1])
        assert bool(torch.isfinite(runs[0][1]).all())


def test_reinforce_agent_loop_with_item_ids(monkeypatch):
    """recnn.nn.Reinforce over item-id batches at 262,144 items with chunking forced on both sides: None on ordinary
    steps, a losses dict exactly at steps 10 and 20, the critic learns every step."""
    monkeypatch.setattr(RF, "_LOGITS_BUDGET_BYTES", 10 * 4096 * 4)
    torch.manual_seed(5)
    S, H, I, N = 52, 64, 262_144, 10
    assert RF._chunk_items(N, I) == 4096
    policy = recnn_b200.nn.DiscreteActor(S, I, H)
    value = recnn_b200.nn.Critic(S, I, H, 54e-2)
    agent = recnn_b200.nn.Reinforce(policy, value).to(torch.device(DEV))
    policy = agent.nets["policy_net"]
    agent.optimizers["policy_optimizer"] = recnn_b200.optim.Adam(policy.parameters(), lr=1e-3)
    agent.optimizers["value_optimizer"] = recnn_b200.optim.Adam(agent.nets["value_net"].parameters(), lr=1e-3)
    rng = np.random.default_rng(8)
    v0 = agent.nets["value_net"].linear1.weight.detach().clone()
    w0 = policy.linear2.weight.detach().clone()
    out = []
    for i in range(21):
        b = ids_batch(rng, N, S, I)
        out.append(agent.update(to_dev(b)))
        agent.step()
        if i == 0:
            assert not torch.equal(v0, agent.nets["value_net"].linear1.weight.detach())
    assert [o is not None for o in out] == [i in (10, 20) for i in range(21)]
    for o in (out[10], out[20]):
        assert set(o) == {"value", "policy", "step"} and np.isfinite(o["value"]) and np.isfinite(o["policy"])
    assert not torch.equal(w0, policy.linear2.weight.detach())
    assert len(policy.rewards) == 0 and len(policy._saved) == 0


def test_reward_line_uses_the_chunked_action_term():
    """reinforce_update's reward = value_net(state, predicted_probs) in item-id mode equals Critic.forward on the dense
    probabilities (eval mode)."""
    rng = np.random.default_rng(2)
    S, H, I, N = 1290, 256, 5000, 64
    algo = make_agent(RO.make_discrete_actor(rng, S, I, H), O.make_critic(rng, S, I, H, 0.3), S, H, I, False)
    state = torch.from_numpy(rng.normal(0, 1, (N, S)).astype(np.float32)).to(DEV)
    probs = algo.nets["policy_net"](state)
    want = algo.nets["value_net"](state, probs)
    got = _ids.critic_value_of_probs(algo.nets["value_net"], state, probs)
    assert float((got - want).abs().max()) <= 1e-5 * float(want.abs().max()) + 1e-7


def test_errors():
    rng = np.random.default_rng(1)
    S, H, I, N = 52, 64, 300, 12
    algo = make_agent(RO.make_discrete_actor(rng, S, I, H), O.make_critic(rng, S, I, H, 0.3), S, H, I, False)
    params = dict(algo.params)
    b = to_dev(ids_batch(rng, N, S, I))
    bad = dict(b, action=b["action"].clone())
    bad["action"][3] = I
    with pytest.raises(IndexError):
        recnn_b200.nn.value_update(bad, params, algo.nets, algo.optimizers, torch.device(DEV), {}, learn=True)
    with pytest.raises(ValueError):
        recnn_b200.nn.value_update(dict(b, action=b["action"].float()), params, algo.nets, algo.optimizers,
                                   torch.device(DEV), {}, learn=True)
    with pytest.raises(ValueError):
        recnn_b200.nn.value_update(dict(b, action=b["action"][:, None].repeat(1, I)), params, algo.nets, algo.optimizers,
                                   torch.device(DEV), {}, learn=True)
    with pytest.raises(ValueError):
        recnn_b200.nn.td3_update(b, params, algo.nets, algo.optimizers, torch.device(DEV), {}, learn=True)
    actor_nets = dict(algo.nets, target_policy_net=recnn_b200.nn.Actor(S, I, H).to(DEV))
    with pytest.raises(ValueError):
        recnn_b200.nn.value_update(b, params, actor_nets, algo.optimizers, torch.device(DEV), {}, learn=True)
    cpu = make_agent(RO.make_discrete_actor(rng, S, I, H), O.make_critic(rng, S, I, H, 0.3), S, H, I, False)
    cpu.nets = {k: v.cpu() for k, v in cpu.nets.items()}
    with pytest.raises(_lib.RecnnError):
        recnn_b200.nn.value_update({k: v.cpu() for k, v in b.items()}, params, cpu.nets, cpu.optimizers,
                                   torch.device("cpu"), {}, learn=True)
    # learn=False: the loss only, and the reference's debug contract (dense target probabilities)
    dbg = {}
    w = algo.nets["value_net"].linear1.weight.detach().clone()
    recnn_b200.nn.value_update(b, params, algo.nets, algo.optimizers, torch.device(DEV), dbg, learn=False)
    assert torch.equal(w, algo.nets["value_net"].linear1.weight.detach())
    assert tuple(dbg["next_action"].shape) == (N, I)
