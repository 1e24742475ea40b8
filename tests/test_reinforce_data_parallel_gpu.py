"""The REINFORCE agent data-parallel over the rows of each batch (recnn_b200.dist.enable_data_parallel on a
DiscreteActor agent), on the GPU.

W > 1 runs as VIRTUAL ranks on one device (tests/_ranks.py): W copies of the public API in one process, each with its
own rows of every batch and a RowParallel over the rank's exchange, attached with dist.data_parallel_in_place.  The
all-reduce is an in-order fp32 sum and the all-gather a rank-order concatenation, as on the peer communicator.  The
API is also checked through a one-rank NCCL group and a real PeerComm; W > 1 processes need W GPUs."""
from __future__ import annotations

import numpy as np
import pytest
import torch

import recnn_b200
from recnn_b200 import _lib
from recnn_b200 import dist as D
from recnn_b200.nn.arena import grad_arena, param_arena
from recnn_b200.nn.update import reinforce as RF
from recnn_b200.nn.update._engine import MASK_KEY
from oracle import reinforce_oracle as RO
from tests import _critic_vocab_oracle as CV
from tests._discrete import PARAMS, critic_case, make_policy, to_dev as _t
from tests._ranks import _copy, bits, exchange, one_rank_group, returned, run_ranks, spawn  # noqa: F401
from tests.test_reinforce_chunked_gpu import REORDER_BAR, unpack

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
L = _lib.lib()
WORLDS = [1, 2, 3, 8]


def plan():
    """This virtual rank's RowParallel over its exchange."""
    ex = exchange()
    return D.RowParallel(None, ex.rank, ex.world, ex)


def rows_of(n, rank, world):
    lo, hi = D.shard_rows(n, rank, world)
    return slice(lo, hi)


# ----------------------------------------------------------------------------- the item-id critic step
def _critic_nets(case, S, H, I, train):
    pp, cp, tcp, _, _ = case
    from tests._cuda import load_net
    policy = make_policy(pp, S, H, I)
    return {"policy_net": policy, "target_policy_net": policy,
            "value_net": load_net(recnn_b200.nn.Critic(S, I, H), cp, DEV).train(train),
            "target_value_net": load_net(recnn_b200.nn.Critic(S, I, H), tcp, DEV)}


def _value_step(nets, batch, masks, rows=slice(None)):
    """(loss, critic) of one value_update over the ``rows`` of an item-id batch, SGD(lr 1e-2)."""
    b = {k: _t(np.ascontiguousarray(v[rows])) for k, v in batch.items()}
    if masks is not None:
        b[MASK_KEY] = [_t(np.ascontiguousarray(m[rows])) for m in masks]
    opt = recnn_b200.optim.SGD(nets["value_net"].parameters(), lr=1e-2)
    loss = recnn_b200.nn.value_update(b, PARAMS, nets, {"value_optimizer": opt}, torch.device(DEV), {}, learn=True)
    return float(loss), nets["value_net"]


def _dp_value_steps(case, S, H, I, world, train, masks, order=None, log=None, patch=None):
    """_value_step on W virtual ranks, each on its rows of the batch and full replicas of the case's nets."""
    full = _critic_nets(case, S, H, I, train)
    batch = case[3]
    n = len(batch["action"])

    def rank(r):
        nets = {k: _copy(v) for k, v in full.items()}
        p = plan()
        if patch is not None:
            patch(r, p)
        D.data_parallel_in_place(nets, p)
        return _value_step(nets, batch, masks, rows_of(n, r, world))
    return run_ranks(world, rank, order=order, log=log)


@pytest.mark.parametrize("train", [False, True], ids=["eval", "masks"])
@pytest.mark.parametrize("world", [2, 3, 8])
def test_critic_step_against_the_oracle(world, train):
    S, H, I, n = 37, 64, 1003, 100
    case = critic_case(S, H, I, n, 11 * world + int(train), 1, train)
    pp, cp, tcp, batch, masks = case
    res = returned(_dp_value_steps(case, S, H, I, world, train, masks))
    losses = [x[0] for x in res]
    assert len({np.float32(x).tobytes() for x in losses}) == 1, losses
    for _, v in res[1:]:
        assert torch.equal(bits(param_arena(v)), bits(param_arena(res[0][1])))
        assert torch.equal(bits(grad_arena(v)), bits(grad_arena(res[0][1])))
    loss1, one = _value_step(_critic_nets(case, S, H, I, train), batch, masks)
    assert losses[0] == pytest.approx(loss1, rel=REORDER_BAR, abs=1e-7)
    g, g1 = grad_arena(res[0][1]), grad_arena(one)
    assert float((g - g1).abs().max()) <= REORDER_BAR * float(g1.abs().max())
    want_loss, want, _ = CV.value_step({"value_net": cp, "target_value_net": tcp, "target_policy_net": pp}, batch, PARAMS,
                                       masks)
    assert losses[0] == pytest.approx(want_loss, rel=2e-5, abs=1e-6)
    got = res[0][1].linear1.weight.grad.double().cpu().numpy()
    assert np.abs(got - want["w1"]).max() <= 1e-4 * np.abs(want["w1"]).max()
    for k, p in (("b1", res[0][1].linear1.bias), ("w2", res[0][1].linear2.weight)):
        assert np.abs(p.grad.double().cpu().numpy() - want[k]).max() <= 1e-4 * np.abs(want[k]).max(), k


@pytest.mark.parametrize("dropout", ["eval", "masks", "philox"])
def test_world1_phases_are_bit_identical_to_the_step(dropout):
    S, H, I, n = 52, 64, 1003, 40
    case = critic_case(S, H, I, n, 5, 1, dropout == "masks")
    masks = case[4]
    train = dropout != "eval"
    torch.manual_seed(3)
    (loss, value), = returned(_dp_value_steps(case, S, H, I, 1, train, masks))
    torch.manual_seed(3)
    loss1, one = _value_step(_critic_nets(case, S, H, I, train), case[3], masks)
    assert np.float32(loss).tobytes() == np.float32(loss1).tobytes()
    assert torch.equal(bits(param_arena(value)), bits(param_arena(one)))
    assert torch.equal(bits(grad_arena(value)), bits(grad_arena(one)))


def test_philox_dropout_follows_the_global_row():
    """Dropout drawn on the device (no masks in the batch): W ranks' rows draw the masks of their global rows, so the
    step matches the single-GPU step within the reordering bar."""
    S, H, I, n = 37, 64, 1003, 100
    case = critic_case(S, H, I, n, 8, 1, False)
    torch.manual_seed(5)
    res = returned(_dp_value_steps(case, S, H, I, 3, True, None))
    torch.manual_seed(5)
    loss1, one = _value_step(_critic_nets(case, S, H, I, True), case[3], None)
    assert res[0][0] == pytest.approx(loss1, rel=REORDER_BAR, abs=1e-7)
    g, g1 = grad_arena(res[0][1]), grad_arena(one)
    assert float((g - g1).abs().max()) <= REORDER_BAR * float(g1.abs().max())


def test_records_out_of_rank_order_and_disagreeing_counts_are_refused():
    S, H, I, n = 37, 64, 1003, 40
    case = critic_case(S, H, I, n, 2, 1, False)
    full = _critic_nets(case, S, H, I, False)
    before = bits(param_arena(full["value_net"]))

    def rank(r, lie):
        nets = {k: _copy(v) for k, v in full.items()}
        p = plan()
        if lie and r == 1:                  # rank 1 counts one row more on rank 2: its n_rows_global disagrees
            true = p.row_counts
            p.row_counts = lambda n_local: [c + (q == 2) for q, c in enumerate(true(n_local))]
        D.data_parallel_in_place(nets, p)
        try:
            _value_step(nets, case[3], None, rows_of(n, r, 3))
        except RuntimeError as exc:
            return exc, bits(param_arena(nets["value_net"]))
        return None, None
    # gather 0 is the row counts, gather 1 the (ids, dz1) records
    for out in (run_ranks(3, lambda r: rank(r, False), order={1: [1, 0, 2]}), run_ranks(3, lambda r: rank(r, True))):
        for exc, arena in out:
            assert isinstance(exc, RuntimeError) and "rank order" in str(exc), exc
            assert torch.equal(arena, before)


def test_out_of_range_id_on_one_rank_raises_everywhere():
    S, H, I, n = 37, 64, 1003, 40
    case = critic_case(S, H, I, n, 4, 1, False)
    batch = dict(case[3])
    batch["action"] = batch["action"].copy()
    batch["action"][D.shard_rows(n, 1, 3)[0]] = I            # rank 1's first row
    before = bits(param_arena(_critic_nets(case, S, H, I, False)["value_net"]))
    full = _critic_nets(case, S, H, I, False)

    def rank(r):
        nets = {k: _copy(v) for k, v in full.items()}
        D.data_parallel_in_place(nets, plan())
        try:
            _value_step(nets, batch, None, rows_of(n, r, 3))
        except IndexError as exc:
            return exc, bits(param_arena(nets["value_net"]))
        return None, None
    for exc, arena in run_ranks(3, rank):
        assert isinstance(exc, IndexError) and "no optimizer step" in str(exc)
        assert torch.equal(arena, before)


def test_beta_out_of_range_id_on_one_rank_takes_no_step():
    S, I, n = 37, 300, 30
    torch.manual_seed(2)
    full = recnn_b200.nn.Beta(S, I).to(DEV)
    rng = np.random.default_rng(1)
    state = _t(rng.normal(0, 1, (n, S)).astype(np.float32))
    ids = rng.integers(0, I, n)
    ids[D.shard_rows(n, 2, 3)[0]] = -1

    def rank(r):
        beta = _copy(full)
        D.data_parallel_in_place({}, plan(), beta)
        before = bits(param_arena(beta))
        try:
            beta(state[rows_of(n, r, 3)], _t(ids[rows_of(n, r, 3)]))
        except IndexError:
            return beta.optim.steps_taken(), torch.equal(before, bits(param_arena(beta)))
        return None
    assert run_ranks(3, rank) == [(0, True)] * 3


def test_exchange_sizes_do_not_grow_with_the_vocabulary():
    S, H, n = 2570, 256, 64
    sizes = []
    for I in (131072, 262144):
        torch.manual_seed(1)
        full = {"policy_net": recnn_b200.nn.DiscreteActor(S, I, H).to(DEV), "value_net": recnn_b200.nn.Critic(S, I, H).to(DEV)}
        full["target_policy_net"], full["target_value_net"] = full["policy_net"], full["value_net"]
        rng = np.random.default_rng(0)
        batch = {"state": rng.normal(0, 1, (n, S)).astype(np.float32),
                 "next_state": rng.normal(0, 1, (n, S)).astype(np.float32), "action": rng.integers(0, I, n),
                 "reward": np.ones(n, np.float32), "done": np.zeros(n, np.float32)}
        log = []

        def rank(r):
            policy = _copy(full["policy_net"])
            nets = {"policy_net": policy, "target_policy_net": policy,
                    "value_net": _copy(full["value_net"]), "target_value_net": _copy(full["value_net"])}
            D.data_parallel_in_place(nets, plan())
            return _value_step(nets, batch, None, rows_of(n, r, 2))[0]
        returned(run_ranks(2, rank, log=log))
        sizes.append([(k, t.numel()) for k, t in log])
        del full
        torch.cuda.empty_cache()
    assert sizes[0] == sizes[1]
    grad = [c for k, c in sizes[0] if k == "all_reduce"]
    assert grad == [H * (((S + 3) // 4 * 4) + H + 3) + 3]


# ----------------------------------------------------------------------------- the policy gradient and the draws
@pytest.mark.parametrize("world", [2, 3, 8])
def test_policy_step_against_the_oracle(world):
    S, H, I, R = 37, 64, 1003, 130
    rng = np.random.default_rng(world)
    p = RO.make_discrete_actor(rng, S, I, H)
    state = rng.normal(0, 1, (R, S)).astype(np.float32)
    blp = np.log(rng.uniform(1e-4, 5e-4, R)).astype(np.float32)
    ret = rng.normal(0, 1, R).astype(np.float32)
    action = rng.integers(0, I, R)
    ret[:] = ret[0]                 # one saved env step per rank: every row has the step's return
    full = make_policy(p, S, H, I)
    for method, fn in ((RO.BASIC, RF.ChooseREINFORCE.basic_reinforce),
                       (RO.TOPK, RF.ChooseREINFORCE.reinforce_with_TopK_correction)):
        def rank(r):
            m = _copy(full)
            D.data_parallel_in_place({"policy_net": m}, plan())
            sl = rows_of(R, r, world)
            m._saved = [{"state": _t(state[sl]), "action": _t(action[sl]),
                         "beta_log_prob": None if method == RO.BASIC else _t(blp[sl]), "K": 10}]
            loss = fn(m, torch.from_numpy(ret[:1]))
            return loss, grad_arena(m).clone()
        res = returned(run_ranks(world, rank))
        assert len({bits(x[0]).item() for x in res}) == 1
        assert all(torch.equal(bits(x[1]), bits(res[0][1])) for x in res)
        want_loss, want, _ = RO.reinforce_policy_grad(p, state, action, None if method == RO.BASIC else blp, ret,
                                                      method, 10)
        assert float(res[0][0]) == pytest.approx(want_loss, rel=2e-4, abs=1e-4 * (1 + abs(want_loss)))
        got = unpack(res[0][1], full)
        for k in ("w1", "b1", "w2", "b2"):
            assert np.abs(got[k].cpu().numpy() - want[k]).max() <= 3e-4 * np.abs(want[k]).max(), (method, k)


def test_draws_at_a_row_offset_are_the_single_gpu_rows():
    n, I = 130, 500
    rng = np.random.default_rng(0)
    probs = torch.softmax(_t(rng.normal(0, 2, (n, I)).astype(np.float32)), 1)
    a1 = torch.empty(n, dtype=torch.int64, device=DEV)
    l1 = torch.empty(n, dtype=torch.float32, device=DEV)
    _lib.check(L.recnn_categorical_sample(probs.data_ptr(), n, I, I, None, 77, 3, a1.data_ptr(), l1.data_ptr(),
                                          _lib.stream_ptr()))
    for lo, hi in [D.shard_rows(n, r, 3) for r in range(3)]:
        a = torch.empty(hi - lo, dtype=torch.int64, device=DEV)
        lp = torch.empty(hi - lo, dtype=torch.float32, device=DEV)
        _lib.check(L.recnn_categorical_sample_at(probs[lo:hi].data_ptr(), hi - lo, I, I, None, 77, 3, lo, a.data_ptr(),
                                                 lp.data_ptr(), _lib.stream_ptr()))
        assert torch.equal(a, a1[lo:hi]) and torch.equal(bits(lp), bits(l1[lo:hi]))


# ----------------------------------------------------------------------------- Reinforce.update() end to end
S_, H_, I_, N_ = 37, 64, 300, 130


def _agent(form, method, opt, seed=7):
    torch.manual_seed(seed)
    policy = recnn_b200.nn.DiscreteActor(S_, I_, H_)
    agent = recnn_b200.nn.Reinforce(policy, recnn_b200.nn.Critic(S_, I_, H_, 54e-2)).to(torch.device(DEV))
    for k in list(agent.optimizers):
        params = agent.nets[k.replace("optimizer", "net")].parameters()
        agent.optimizers[k] = (recnn_b200.optim.Adam(params, lr=1e-3) if opt == "adam"
                               else torch.optim.Adam(params, lr=1e-3))
    agent.params["policy_step"] = 10
    beta = None
    if method == "topk":
        beta = recnn_b200.nn.Beta(S_, I_).to(DEV)
        beta.optim = recnn_b200.optim.RAdam(beta.net.parameters(), lr=1e-2, weight_decay=1e-5)
        agent.params["reinforce"] = recnn_b200.nn.ChooseREINFORCE(
            recnn_b200.nn.ChooseREINFORCE.reinforce_with_TopK_correction)
    return agent, beta


def _wire_beta(agent, beta):
    if beta is None:
        return
    pol = agent.nets["policy_net"]

    def select(state, action, K, writer, step, **kwargs):
        return pol._select_action_with_TopK_correction(state, beta.forward, action, K=K, writer=writer, step=step)
    pol.select_action = select


def _batch(step, form):
    rng = np.random.default_rng(100 + step)
    ids = rng.integers(0, I_, N_)
    action = ids if form == "ids" else np.eye(I_, dtype=np.float32)[ids]
    return {"state": rng.normal(0, 1, (N_, S_)).astype(np.float32), "action": action,
            "reward": (rng.integers(1, 6, N_) - 3).astype(np.float32),
            "next_state": rng.normal(0, 1, (N_, S_)).astype(np.float32),
            "done": (rng.random(N_) < 0.1).astype(np.float32)}


def _snapshot(agent, beta):
    out = [bits(param_arena(agent.nets[k])) for k in sorted(agent.nets)]
    opts = [agent.optimizers[k] for k in sorted(agent.optimizers)] + ([beta.optim] if beta is not None else [])
    for o in opts:
        if isinstance(o, recnn_b200.optim._ArenaOptimizer):
            out += [bits(t) for t in (o._m, o._v) if t is not None]
        else:
            out += [bits(v) for st in o.state.values() for v in st.values() if torch.is_tensor(v) and v.dim() > 0]
    if beta is not None:
        out.append(bits(param_arena(beta)))
    return out


def _run(agent, beta, form, rows=slice(None), steps=21):
    _wire_beta(agent, beta)
    trace = []
    for step in range(steps):
        b = {k: torch.from_numpy(np.ascontiguousarray(v[rows])) for k, v in _batch(step, form).items()}
        torch.manual_seed(1000 + step)
        losses = agent.update(b)
        agent.step()
        pol = agent.nets["policy_net"]
        saved = torch.cat([r["action"] for r in pol._saved]).cpu() if pol._saved else None
        trace.append((losses, _snapshot(agent, beta), saved))
    return trace


def _dp_run(world, form, method, opt, steps=21):
    def rank(r):
        agent, beta = _agent(form, method, opt)
        D.data_parallel_in_place(agent.nets, plan(), beta, agent.optimizers)
        return _run(agent, beta, form, rows_of(N_, r, world), steps)
    return returned(run_ranks(world, rank))


CASES = [("ids", "basic", "adam"), ("onehot", "basic", "adam"), ("ids", "topk", "adam"), ("onehot", "topk", "adam")]


@pytest.mark.parametrize("form,method,opt", CASES + [("ids", "topk", "torch")], ids="-".join)
@pytest.mark.parametrize("world", WORLDS)
def test_reinforce_updates(world, form, method, opt):
    if opt == "torch" and world not in (1, 3):
        pytest.skip("the torch-optimizer variant runs at W = 1 and 3")
    res = _dp_run(world, form, method, opt)
    policy_steps = 0
    for step in range(21):
        ref = res[0][step]
        policy_steps += ref[0] is not None
        for other in res[1:]:
            assert other[step][0] == ref[0], step
            assert all(torch.equal(x, y) for x, y in zip(other[step][1], ref[1])), step
    assert policy_steps == 2
    agent, beta = _agent(form, method, opt)
    one = _run(agent, beta, form)
    if world == 1:
        for step in range(21):
            assert res[0][step][0] == one[step][0], step
            assert all(torch.equal(x, y) for x, y in zip(res[0][step][1], one[step][1])), step
            assert (res[0][step][2] is None) == (one[step][2] is None)
            if one[step][2] is not None:
                assert torch.equal(res[0][step][2], one[step][2]), step
    else:
        assert torch.equal(torch.cat([r[0][2] for r in res]), one[0][2])


def test_enable_data_parallel_world1_equals_unsharded(one_rank_group):
    plain, plain_beta = _agent("ids", "topk", "adam")
    dp, dp_beta = _agent("ids", "topk", "adam")
    D.enable_data_parallel(dp, beta=dp_beta)
    p = D.row_parallel_of(dp.nets["policy_net"])
    assert isinstance(p.comm, D.PeerComm) and p.world == 1 and D.row_parallel_of(dp_beta) is p
    a, b = _run(plain, plain_beta, "ids", steps=11), _run(dp, dp_beta, "ids", steps=11)
    for x, y in zip(a, b):
        assert x[0] == y[0]
        assert all(torch.equal(u, v) for u, v in zip(x[1], y[1]))
    # state_dict round trip of a replica: the unsharded layout
    assert set(dp.nets["value_net"].state_dict()) == set(plain.nets["value_net"].state_dict())
    p.comm.close()


def _mp_worker(rank, world, port, q):
    import os
    import torch.distributed as dist
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    try:
        global DEV
        DEV = "cuda:%d" % rank
        agent, beta = _agent("ids", "topk", "adam")
        D.enable_data_parallel(agent, beta=beta)
        trace = _run(agent, beta, "ids", rows_of(N_, rank, world), steps=11)
        q.put((rank, [t[0] for t in trace], [[x.tolist() for x in t[1]] for t in trace]))
        D.row_parallel_of(agent.nets["policy_net"]).comm.close()
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 4, 8])
def test_multi_process(world):
    if torch.cuda.device_count() < world:
        pytest.skip("needs %d GPUs" % world)
    out = sorted(spawn(_mp_worker, world))
    for _, losses, arenas in out[1:]:
        assert losses == out[0][1] and arenas == out[0][2]
