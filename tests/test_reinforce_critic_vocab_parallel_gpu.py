"""The item-id REINFORCE critic sharded over the item vocabulary, on the GPU.

As in test_reinforce_vocab_parallel_gpu.py, the maths is checked with VIRTUAL ranks on one device: the three C phases of
W shards run in one process, the all-gather is stood in for by concatenating the ranks' records in rank order and the
all-reduce of the [2, N, H] terms by an in-order fp32 sum.  The Python API is checked at world 1 through a one-rank
NCCL group against an unsharded twin, bit for bit; W > 1 processes need W GPUs."""
from __future__ import annotations

import gc
import os

import numpy as np
import pytest
import torch

import recnn_b200
from recnn_b200 import _lib
from recnn_b200 import dist as D
from recnn_b200.nn.arena import param_arena, grad_arena
from recnn_b200.nn.update import reinforce as RF
from oracle import recnn_oracle as O
from oracle import reinforce_oracle as RO
from tests import _critic_vocab_oracle as CV
from tests._cuda import load_net
from tests._discrete import (PARAMS, critic_case as _case, critic_ranks as _ranks, make_policy,
                             to_dev as _t)
from tests.test_reinforce_chunked_gpu import REORDER_BAR

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
L = _lib.lib()
# (S, H, items, rows, chunk): S % 4 == 0 and S % 4 != 0; local blocks chunked with a ragged last chunk (W = 1, 3) and
# narrower than one chunk (W = 8)
SHAPES = [(52, 64, 1003, 40, 128), (37, 32, 2000, 33, 256)]


def run_phases(ranks, order=None):
    """begin on every rank, the all-gather (records concatenated in ``order``), merge, the in-order fp32 sum of the
    terms, end.  Returns the summed terms."""
    st = _lib.stream_ptr()
    n = ranks[0].n
    recs = []
    for rk in ranks:
        recs.append(torch.empty(L.recnn_vocab_record_floats(n), device=DEV))
        _lib.check(L.recnn_discrete_value_shard_begin(rk.args, rk.shard, recs[-1].data_ptr(), st))
    gathered = torch.cat([recs[q] for q in (order or range(len(ranks)))])
    terms = []
    for rk in ranks:
        terms.append(torch.empty(2 * n * rk.args.dims.hidden, device=DEV))
        _lib.check(L.recnn_discrete_value_shard_merge(rk.args, rk.shard, gathered.data_ptr(), terms[-1].data_ptr(), st))
    acc = terms[0].clone()
    for t in terms[1:]:
        acc += t
    for rk in ranks:
        _lib.check(L.recnn_discrete_value_shard_end(rk.args, rk.shard, acc.data_ptr(), st))
    torch.cuda.synchronize()
    return acc


def _unsharded(pp, cp, tcp, S, H, I, chunk, batch, masks, lr=1e-2):
    (rk,), _, _ = _ranks(pp, cp, tcp, S, H, I, 1, chunk, batch, masks, lr)
    _lib.check(L.recnn_discrete_value_step(rk.args, _lib.stream_ptr()))
    torch.cuda.synchronize()
    return rk


def _bits(t):
    return t.detach().contiguous().view(torch.int32)


def _blocks(m, S):
    """(replicated tensors, action block) of a critic's parameters and gradients."""
    w, g = m.linear1.weight.detach(), m.linear1.weight.grad
    rest = list(m.parameters())[1:]
    rep = [w[:, :S], g[:, :S]] + [p.detach() for p in rest] + [p.grad for p in rest]
    return rep, w[:, S:], g[:, S:]


@pytest.mark.parametrize("train", [False, True], ids=["eval", "masks"])
@pytest.mark.parametrize("world", [1, 2, 3, 8])
@pytest.mark.parametrize("S,H,I,n,chunk", SHAPES)
def test_virtual_ranks(S, H, I, n, chunk, world, train):
    pp, cp, tcp, batch, masks = _case(S, H, I, n, S + I + world + int(train), world, train)
    ranks, dev_batch, _ = _ranks(pp, cp, tcp, S, H, I, world, chunk, batch, masks)
    one = _unsharded(pp, cp, tcp, S, H, I, chunk, batch, masks)
    terms = run_phases(ranks)
    # the loss and every replicated block (gradient and stepped weights) have the same bits on every rank
    assert all(rk.loss_bits() == ranks[0].loss_bits() for rk in ranks)
    assert ranks[0].loss_bits()[1] == 0
    rep0 = _blocks(ranks[0].value, S)[0]
    for rk in ranks[1:]:
        for x, y in zip(_blocks(rk.value, S)[0], rep0):
            assert torch.equal(_bits(x), _bits(y))
    # the summed online action term is the unsharded gather bit for bit (exactly one rank contributes to each row)
    add = terms[n * H:].view(n, H)
    want_add = _t(cp["w1"])[:, S + dev_batch["action"]].T
    assert torch.equal(_bits(add), _bits(want_add))
    # against the unsharded CUDA step: loss and replicated blocks within the reordering bar, the action block too
    loss, loss1 = float(ranks[0].losses[0]), float(one.losses[0])
    assert loss == pytest.approx(loss1, rel=REORDER_BAR, abs=1e-7)
    rep1, _, g1 = _blocks(one.value, S)
    for x, y in zip(rep0, rep1):
        assert float((x - y).abs().max()) <= REORDER_BAR * max(float(y.abs().max()), 1e-30)
    gblock = torch.cat([_blocks(rk.value, S)[2] for rk in ranks], 1)
    assert float((gblock - g1).abs().max()) <= REORDER_BAR * float(g1.abs().max())
    wblock = torch.cat([_blocks(rk.value, S)[1] for rk in ranks], 1)
    w1 = one.value.linear1.weight.detach()[:, S:]
    assert float((wblock - w1).abs().max()) <= REORDER_BAR * float(w1.abs().max())
    # against the float64 oracle at the item-id critic's bars
    want_loss, want, _ = CV.value_step({"value_net": cp, "target_value_net": tcp, "target_policy_net": pp}, batch, PARAMS,
                                       masks)
    assert loss == pytest.approx(want_loss, rel=2e-5, abs=1e-6)
    got_gw1 = torch.cat([ranks[0].value.linear1.weight.grad[:, :S], gblock], 1).double().cpu().numpy()
    scale = np.abs(want["w1"]).max()
    assert np.abs(got_gw1 - want["w1"]).max() <= 1e-4 * scale
    unselected = torch.from_numpy(np.setdiff1d(np.arange(I), batch["action"])).to(DEV)
    assert int((gblock[:, unselected] != 0).sum()) == 0


@pytest.mark.parametrize("S,H,I,n,chunk", SHAPES)
def test_world1_phases_are_bit_identical_to_the_step(S, H, I, n, chunk):
    for train in (False, True):
        pp, cp, tcp, batch, masks = _case(S, H, I, n, 5 * S, 1, train)
        ranks, _, _ = _ranks(pp, cp, tcp, S, H, I, 1, chunk, batch, masks)
        one = _unsharded(pp, cp, tcp, S, H, I, chunk, batch, masks)
        run_phases(ranks)
        assert ranks[0].loss_bits() == one.loss_bits()
        assert torch.equal(_bits(param_arena(ranks[0].value)), _bits(param_arena(one.value)))
        assert torch.equal(_bits(grad_arena(ranks[0].value)), _bits(grad_arena(one.value)))


def test_records_out_of_rank_order_are_flagged():
    S, H, I, n, chunk = SHAPES[0]
    pp, cp, tcp, batch, masks = _case(S, H, I, n, 3, 3, False)
    ranks, _, _ = _ranks(pp, cp, tcp, S, H, I, 3, chunk, batch, masks)
    run_phases(ranks, order=[1, 0, 2])
    assert all(rk.loss_bits()[1] & 2 for rk in ranks)


# ----------------------------------------------------------------------------- the Python API at world 1
@pytest.fixture
def one_rank_group(tmp_path):
    import torch.distributed as dist
    torch.cuda.set_device(0)
    dist.init_process_group("nccl", init_method="file://" + str(tmp_path / "pg"), rank=0, world_size=1,
                            device_id=torch.device(DEV))
    yield
    dist.destroy_process_group()


def _twins(S, H, I, variant):
    agents = []
    for _ in range(2):
        torch.manual_seed(17)
        agent = recnn_b200.nn.Reinforce(recnn_b200.nn.DiscreteActor(S, I, H), recnn_b200.nn.Critic(S, I, H, 0.3))
        agent = agent.to(torch.device(DEV))
        agent.params["policy_step"] = 4
        nets = agent.nets
        if variant == "adam":
            agent.optimizers = {"policy_optimizer": recnn_b200.optim.Adam(nets["policy_net"].parameters(), lr=1e-3),
                                "value_optimizer": recnn_b200.optim.Adam(nets["value_net"].parameters(), lr=1e-3)}
        else:
            agent.optimizers = {"policy_optimizer": torch.optim.SGD(nets["policy_net"].parameters(), lr=1e-2),
                                "value_optimizer": torch.optim.SGD(nets["value_net"].parameters(), lr=1e-2)}
        agents.append(agent)
    D.enable_vocab_parallel(agents[1])
    return agents


def _ids_batch(rng, N, S, I):
    a = rng.integers(0, I, N)
    a[:N // 4] = a[N // 4:N // 2]
    return {"state": _t(rng.normal(0, 1, (N, S)).astype(np.float32)),
            "next_state": _t(rng.normal(0, 1, (N, S)).astype(np.float32)), "action": _t(a),
            "reward": _t((rng.integers(1, 6, N) - 3).astype(np.float32)),
            "done": _t((rng.random(N) < 0.1).astype(np.float32))}


def _same_arenas(a, b):
    for k in a.nets:
        assert torch.equal(_bits(param_arena(a.nets[k])), _bits(param_arena(b.nets[k]))), k
    for k in ("policy_net", "value_net"):
        assert torch.equal(_bits(grad_arena(a.nets[k])), _bits(grad_arena(b.nets[k]))), k


@pytest.mark.parametrize("variant", ["adam", "torch_sgd"])
def test_python_api_world1_equals_unsharded(one_rank_group, variant):
    """A Reinforce agent over item-id batches, 20 update() calls (policy steps at 4, 8, ..., 16), against its
    unsharded twin: losses, every parameter arena and both gradient arenas bit for bit."""
    S, H, I, N = 52, 64, 1003, 16
    plain, shard = _twins(S, H, I, variant)
    vp = shard.nets["policy_net"].__dict__["_recnn_vp"]
    assert all(shard.nets[k].__dict__["_recnn_vp"] is vp for k in shard.nets)
    assert (vp.lo, vp.hi, vp.world) == (0, I, 1)
    if variant == "adam":
        assert all(isinstance(o, recnn_b200.optim.Adam) for o in shard.optimizers.values())
        assert shard.optimizers["value_optimizer"].param_groups[0]["lr"] == 1e-3
    rng = np.random.default_rng(4)
    policy_steps = 0
    for i in range(20):
        b = _ids_batch(rng, N, S, I)
        outs = []
        for agent in (plain, shard):
            torch.manual_seed(1000 + i)
            outs.append(agent.update(b))
            agent.step()
        assert outs[0] == outs[1], i
        policy_steps += outs[0] is not None
        _same_arenas(plain, shard)
    assert policy_steps == 4
    # learn=False: the loss and the debug contract (the rank's column block, here all of it)
    losses = []
    for agent in (plain, shard):
        torch.manual_seed(7)
        agent.debug = {}
        losses.append(float(recnn_b200.nn.value_update(b, agent.params, agent.nets, agent.optimizers, torch.device(DEV),
                                                       agent.debug, learn=False)))
    assert losses[0] == losses[1]
    assert torch.equal(plain.debug["next_action"], shard.debug["next_action"])
    # an id >= num_items: IndexError on both, and the update applied with the offending rows' action term set to zero
    bad = dict(b, action=b["action"].clone())
    bad["action"][[2, 9]] = I
    for agent in (plain, shard):
        torch.manual_seed(8)
        with pytest.raises(IndexError):
            recnn_b200.nn.value_update(bad, agent.params, agent.nets, agent.optimizers, torch.device(DEV), {},
                                       learn=True)
    _same_arenas(plain, shard)
    # a dense action on the sharded agent
    with pytest.raises(RuntimeError, match="ChooseREINFORCE"):
        shard.update(dict(b, action=torch.zeros(N, I, device=DEV)))
    with pytest.raises(RuntimeError):
        recnn_b200.nn.value_update(dict(b, action=torch.zeros(N, I, device=DEV)), shard.params, shard.nets,
                                   shard.optimizers, torch.device(DEV), {}, learn=True)
    vp.comm.close()


# ----------------------------------------------------------------------------- one rank's share of configs[4]
def test_config4_rank_share_memory_is_bounded():
    """S 2570 / H 256, 1M items over 8 ranks (125,000 local), 16,384 rows: the three phases of the last virtual rank,
    with every other rank's record standing in as a copy of this one's.  The extra memory is the workspace, W records and
    the [2, N, H] terms, far below one dense [N, num_items] action (68.7 GB)."""
    S, H, I, world, N = 2570, 256, 1_000_000, 8, 16_384
    lo, hi = D.vocab_shard(I, world - 1, world)
    torch.manual_seed(3)
    with torch.device(DEV):
        policy = recnn_b200.nn.DiscreteActor(S, hi - lo, H)
        value, target = recnn_b200.nn.Critic(S, hi - lo, H, 3e-3), recnn_b200.nn.Critic(S, hi - lo, H, 3e-3)
        b = {"state": torch.randn(N, S), "next_state": torch.randn(N, S), "action": torch.randint(0, I, (N,)),
             "reward": torch.randn(N), "done": torch.zeros(N)}
    b["action"][:3] = torch.tensor([lo, hi - 1, lo + 1])
    chunk = RF._chunk_items(N, hi - lo)
    opt = recnn_b200.optim.SGD(value.parameters(), lr=1e-3).bind(value)
    a = _lib.DiscreteValueArgs()
    a.dims, a.policy_dims = _lib.Dims(S, hi - lo, H, 0), policy.dims
    a.learn, a.chunk_items, a.n_rows = 1, chunk, N
    a.state, a.next_state, a.action = b["state"].data_ptr(), b["next_state"].data_ptr(), b["action"].data_ptr()
    a.reward, a.done = b["reward"].data_ptr(), b["done"].data_ptr()
    a.value = opt.c_net(value)
    a.target_value = _lib.Net(param_arena(target).data_ptr(), None, None, None, None, None)
    a.target_policy = param_arena(policy).data_ptr()
    a.value_optim = opt.c_optim()
    a.gamma, a.min_value, a.max_value = 0.99, -10.0, 10.0
    rng_step, losses = torch.zeros(1, dtype=torch.int64, device=DEV), torch.zeros(8, device=DEV)
    a.rng_step, a.losses = rng_step.data_ptr(), losses.data_ptr()
    vs = _lib.VocabShard(lo, I, world - 1, world)
    st = _lib.stream_ptr()
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    nbytes = L.recnn_discrete_value_workspace_bytes(a.dims, a.policy_dims, N, chunk)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=DEV)
    a.workspace, a.workspace_bytes = ws.data_ptr(), nbytes
    rec = torch.empty(L.recnn_vocab_record_floats(N), device=DEV)
    _lib.check(L.recnn_discrete_value_shard_begin(a, vs, rec.data_ptr(), st))
    gathered = rec.repeat(world)
    hdr = gathered.view(world, -1)[:, :4].view(torch.int32)
    for q in range(world):
        hdr[q, :2] = torch.tensor(D.vocab_shard(I, q, world), dtype=torch.int32)
    terms = torch.empty(2 * N * H, device=DEV)
    _lib.check(L.recnn_discrete_value_shard_merge(a, vs, gathered.data_ptr(), terms.data_ptr(), st))
    _lib.check(L.recnn_discrete_value_shard_end(a, vs, terms.data_ptr(), st))
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    print("configs[4] rank share: chunk %d, workspace %.3f GB, terms %.1f MB, peak extra %.3f GB"
          % (chunk, nbytes / 1e9, terms.numel() * 4 / 1e6, peak / 1e9))
    assert losses.view(torch.int32)[4].item() == 0
    assert np.isfinite(float(losses[0]))
    assert peak <= nbytes + (world + 1) * rec.numel() * 4 + terms.numel() * 4 + (64 << 20)
    assert peak < N * I * 4 / 16


# ----------------------------------------------------------------------------- W > 1 processes
def _agent(S, H, I, seed=31):
    torch.manual_seed(seed)
    agent = recnn_b200.nn.Reinforce(recnn_b200.nn.DiscreteActor(S, I, H), recnn_b200.nn.Critic(S, I, H, 0.3))
    agent.params["policy_step"] = 1
    agent.optimizers = {"policy_optimizer": recnn_b200.optim.SGD(agent.nets["policy_net"].parameters(), lr=1e-2),
                        "value_optimizer": recnn_b200.optim.SGD(agent.nets["value_net"].parameters(), lr=1e-2)}
    return agent


def _mp_batches(S, I, N=24):
    rng = np.random.default_rng(12)
    out = []
    for _ in range(2):
        a = rng.integers(0, I, N)
        a[:N // 4] = a[N // 4:N // 2]
        out.append({"state": rng.normal(0, 1, (N, S)).astype(np.float32),
                    "next_state": rng.normal(0, 1, (N, S)).astype(np.float32), "action": a,
                    "reward": (rng.integers(1, 6, N) - 3).astype(np.float32),
                    "done": (rng.random(N) < 0.1).astype(np.float32)})
    return out


def _run_agent(agent, dev):
    outs = []
    for i, b in enumerate(_mp_batches(52, 1003)):
        torch.manual_seed(50 + i)
        outs.append(agent.update({k: torch.from_numpy(v).to(dev) for k, v in b.items()}))
        agent.step()
    return outs


def _mp_worker(rank, world, port, q):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    try:
        agent = _agent(52, 64, 1003).to(dev)
        D.enable_vocab_parallel(agent)
        outs = _run_agent(agent, dev)
        vp = agent.nets["value_net"].__dict__["_recnn_vp"]
        v = agent.nets["value_net"]
        q.put((rank, {"outs": outs, "lo": vp.lo, "hi": vp.hi,
                      "rep": [p.detach().cpu().numpy() for p in list(v.parameters())[1:]]
                      + [v.linear1.weight.detach()[:, :52].cpu().numpy(),
                         agent.nets["policy_net"].linear1.weight.detach().cpu().numpy()],
                      "block": v.linear1.weight.detach()[:, 52:].cpu().numpy()}))
        torch.cuda.synchronize()
        vp.comm.close()
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 4, 8])
def test_multi_process_equals_unsharded(world):
    if torch.cuda.device_count() < world:
        pytest.skip("needs %d GPUs" % world)
    import socket
    import torch.multiprocessing as mp
    s = socket.socket(); s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]; s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_mp_worker, args=(r, world, port, q)) for r in range(world)]
    for pr in procs:
        pr.start()
    res = dict(q.get(timeout=300) for _ in range(world))
    for pr in procs:
        pr.join(timeout=60)
        assert pr.exitcode == 0
    full = _agent(52, 64, 1003).to(torch.device(DEV))
    want = _run_agent(full, torch.device(DEV))
    for r in range(world):
        assert res[r]["outs"] == res[0]["outs"]
        for x, y in zip(res[r]["rep"], res[0]["rep"]):
            assert np.array_equal(x.view(np.int32), y.view(np.int32))
    got, ref = res[0]["outs"][1], want[1]
    for k in ("value", "policy"):
        assert got[k] == pytest.approx(ref[k], rel=REORDER_BAR, abs=1e-7), k
    block = np.concatenate([res[r]["block"] for r in range(world)], 1)
    wref = full.nets["value_net"].linear1.weight.detach()[:, 52:].cpu().numpy()
    assert np.abs(block - wref).max() <= REORDER_BAR * np.abs(wref).max()
