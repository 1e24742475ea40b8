"""Full checkpoints of a vocabulary-parallel REINFORCE agent and its β on the GPU: the gathered state of a trained
world-1 agent against its unsharded twin's state_dicts bit for bit, resuming from it (unsharded and sharded), serving
the gathered policy's top-k on one GPU, virtual ranks 2 / 3 / 8 on one device (load path, then the gather's transport
halves in process), the device memory of the gather, and W = 2 / 4 / 8 processes where that many GPUs exist."""
from __future__ import annotations

import gc
import os

import numpy as np
import pytest
import torch

import recnn_b200
from recnn_b200 import dist as D
from recnn_b200.nn.arena import param_arena
from tests._ranks import one_rank_group, spawn  # noqa: F401
from tests.test_beta_vocab_parallel_gpu import _notebook_agent
from tests.test_vocab_checkpoint_host import _full_state, _same

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
S, H, ITEMS, N = 37, 64, 1003, 10              # the shapes _notebook_agent builds
SOURCE = {"pi": "pi", "beta": "beta"}


def _batch(step):
    rng = np.random.default_rng(100 + step)
    return {"state": torch.from_numpy(rng.normal(0, 1, (N, S)).astype(np.float32)),
            "action": torch.from_numpy(rng.integers(0, ITEMS, N)),
            "reward": torch.from_numpy(rng.integers(1, 6, N).astype(np.float32) - 3),
            "next_state": torch.from_numpy(rng.normal(0, 1, (N, S)).astype(np.float32)),
            "done": torch.from_numpy((rng.random(N) < 0.1).astype(np.float32)),
            # the critic's dropout masks from the batch: drawn ones follow a per-engine counter no checkpoint carries
            "dropout_masks": [torch.from_numpy((rng.random((N, H)) < 0.5).astype(np.uint8)) for _ in range(2)]}


def _run(agent, steps):
    """``steps`` more updates from the agent's step counter; the losses of the policy steps."""
    losses = []
    for _ in range(steps):
        step = agent._step
        torch.manual_seed(1000 + step)          # the same dropout masks and draws for every agent
        losses.append(agent.update(_batch(step)))
        agent.step()
    return losses


def _agent(shard, group=None):
    agent, beta, _ = _notebook_agent(SOURCE)
    agent.params["policy_step"] = 3             # policy updates at steps 3, 6, 9, 12
    if shard:
        D.enable_vocab_parallel(agent, group=group, beta=beta)
    return agent, beta


def _trained(shard, group=None):
    agent, beta = _agent(shard, group)
    _run(agent, 7)                              # two policy updates, the checkpoint right after the second
    return agent, beta


def _close(agent):
    vp = agent.nets["policy_net"].__dict__.get("_recnn_vp")
    if vp is not None and vp.comm is not None:
        torch.cuda.synchronize()
        vp.comm.close()


def _on_host(x):
    if torch.is_tensor(x):
        return x.device.type == "cpu"
    if isinstance(x, dict):
        return all(_on_host(v) for v in x.values())
    if isinstance(x, (list, tuple)):
        return all(_on_host(v) for v in x)
    return True


def test_world1_gather_equals_the_unsharded_twin(one_rank_group):
    plain, plain_beta = _trained(False)
    shard, shard_beta = _trained(True)
    got = D.gather_vocab_parallel_state(shard, beta=shard_beta)
    assert _on_host(got)
    assert got["optimizers"]["policy_optimizer"]["recnn_arenas"]["t"] == 2
    assert got["beta"]["optim"]["recnn_arenas"]["t"] == 7
    _same(got, _full_state(plain, plain_beta))
    _close(shard)


def _load_unsharded(agent, beta, ckpt):
    for k, net in agent.nets.items():
        net.load_state_dict(ckpt["nets"][k])
    for k, opt in agent.optimizers.items():
        opt.load_state_dict(ckpt["optimizers"][k])
    beta.load_state_dict(ckpt["beta"]["net"])
    beta.optim.load_state_dict(ckpt["beta"]["optim"])


def test_world1_resume_continues_the_uninterrupted_run(one_rank_group):
    ref, ref_beta = _trained(True)
    ckpt = D.gather_vocab_parallel_state(ref, beta=ref_beta)
    resumed = []
    for shard in (False, True):
        agent, beta = _agent(shard)
        if shard:
            D.load_vocab_parallel_state(agent, ckpt, beta=beta)
        else:
            _load_unsharded(agent, beta, ckpt)
        # not part of a checkpoint, as for the unsharded state_dict: the update counter and the policy's draw counter
        agent._step, agent.nets["policy_net"]._draws = ref._step, ref.nets["policy_net"]._draws
        resumed.append((agent, beta))
    want = _run(ref, 6)
    assert sum(x is not None for x in want) == 2
    for agent, beta in resumed:
        assert _run(agent, 6) == want
    final = D.gather_vocab_parallel_state(ref, beta=ref_beta)
    _same(_full_state(*resumed[0]), final)
    _same(D.gather_vocab_parallel_state(resumed[1][0], beta=resumed[1][1]), final)
    for agent, _ in [(ref, None)] + resumed:
        _close(agent)


def test_serving_the_gathered_policy_on_one_gpu(one_rank_group):
    shard, shard_beta = _trained(True)
    ckpt = D.gather_vocab_parallel_state(shard.nets["policy_net"])
    solo = recnn_b200.nn.DiscreteActor(S, ITEMS, H).to(DEV)
    solo.load_state_dict(ckpt["nets"]["policy_net"])
    state = torch.randn(50, S, device=DEV)
    for k in (1, 10, 64):
        v1, i1 = solo.topk(state, k)
        v2, i2 = shard.nets["policy_net"].topk(state, k)
        assert torch.equal(i1, i2) and torch.equal(v1, v2), k
    _close(shard)


@pytest.mark.parametrize("world", [2, 3, 8])
def test_virtual_ranks_on_one_device(one_rank_group, monkeypatch, world):
    """A trained agent's full state into W local blocks through the load path, back through the transport halves with
    an in-process list."""
    monkeypatch.setattr(D, "_SLICE_FLOATS", 4096)        # several slices per block
    plain, plain_beta = _trained(False)
    full = _full_state(plain, plain_beta)
    ranks = []
    for r in range(world):
        lo, hi = D.vocab_shard(ITEMS, r, world)
        agent = recnn_b200.nn.Reinforce(recnn_b200.nn.DiscreteActor(S, ITEMS, H).to(DEV),
                                        recnn_b200.nn.Critic(S, ITEMS, H).to(DEV)).to(torch.device(DEV))
        beta = recnn_b200.nn.Beta(S, ITEMS).to(DEV)
        D.shard_in_place(agent.nets, D.VocabParallel(lo, hi, ITEMS, None, r, world, None), beta, agent.optimizers)
        D.load_vocab_parallel_state(agent, full, beta=beta)
        assert torch.equal(beta.net[0].weight, plain_beta.net[0].weight[lo:hi])
        assert torch.equal(agent.nets["target_value_net"].linear1.weight[:, S:],
                           plain.nets["target_value_net"].linear1.weight[:, S + lo:S + hi])
        nets, opts, _ = D._checkpoint_parts(agent, beta)
        ranks.append(D._gather_begin(nets, opts, ITEMS, r == 0) + (hi - lo,))
    leaves, _, out, _ = ranks[0]
    D._copy_shared(leaves)
    for q, (q_leaves, _, _, n) in enumerate(ranks):
        lo, hi = D.vocab_shard(ITEMS, q, world)
        for v, s in zip(D._inbox(leaves, lo, hi), list(D._outbox(q_leaves, n))):
            v.copy_(s)
    _same(out, full)


def test_gather_device_memory(one_rank_group):
    """S 1290 x 262,144 items, H 256, Ranger and β RAdam: the gather adds at most one slice (+ 64 MB) to the resident
    arenas."""
    S_, I_, H_ = 1290, 262144, 256
    torch.manual_seed(0)
    with torch.device(DEV):
        agent = recnn_b200.nn.Reinforce(recnn_b200.nn.DiscreteActor(S_, I_, H_), recnn_b200.nn.Critic(S_, I_, H_))
        beta = recnn_b200.nn.Beta(S_, I_)
    agent.to(torch.device(DEV))
    D.enable_vocab_parallel(agent, beta=beta)
    owners = {"policy_optimizer": "policy_net", "value_optimizer": "value_net"}
    for k, opt in agent.optimizers.items():             # arenas as after a step
        opt.c_net(agent.nets[owners[k]])
        opt._t.fill_(1)
    beta.optim.c_net(beta)
    beta.optim._t.fill_(1)
    gc.collect()
    torch.cuda.synchronize()
    resident = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    ckpt = D.gather_vocab_parallel_state(agent, beta=beta)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated()
    print("resident %.2f GB, gather peak above it %.1f MB" % (resident / 1e9, (peak - resident) / 2 ** 20))
    assert peak <= resident + D._SLICE_FLOATS * 4 + (64 << 20)
    assert torch.equal(ckpt["beta"]["net"]["net.0.weight"][-3:], beta.net[0].weight[-3:].cpu())
    _close(agent)


# ----------------------------------------------------------------------------------------------------- W > 1 processes
def _mp_worker(rank, world, port, path, q):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    from tests import test_beta_vocab_parallel_gpu as TB
    global DEV
    DEV = TB.DEV = "cuda:%d" % rank                   # _notebook_agent builds on TB.DEV
    try:
        agent, beta = _trained(True)
        draws = agent.nets["policy_net"]._draws
        ckpt = D.gather_vocab_parallel_state(agent, beta=beta)
        if rank == 0:
            torch.save(ckpt, path)
        _close(agent)
        dist.barrier()
        # resume at another world size: the first half of the ranks, in a group of their own
        half = dist.new_group(list(range(world // 2)))
        res = None
        if rank < world // 2:
            agent, beta = _agent(True, group=half)
            D.load_vocab_parallel_state(agent, torch.load(path, weights_only=False), beta=beta)
            agent._step, agent.nets["policy_net"]._draws = 7, draws
            losses = _run(agent, 6)
            res = (losses, D.gather_vocab_parallel_state(agent, beta=beta))
            _close(agent)
        if rank == 0:
            q.put((ckpt, res))
        dist.barrier()
    finally:
        dist.destroy_process_group()


def _near(got, want, atol):
    if torch.is_tensor(want):
        torch.testing.assert_close(got.float(), want.detach().cpu().float(), rtol=1e-4, atol=atol)
    elif isinstance(want, dict):
        for k in want:
            if k not in ("t", "step", "param_groups"):
                _near(got[k], want[k], atol)


@pytest.mark.parametrize("world", [2, 4, 8])
def test_multi_process_gather_and_resume_at_another_world_size(tmp_path, world):
    if torch.cuda.device_count() < world:
        pytest.skip("needs %d GPUs" % world)
    (ckpt, (losses, resumed)), = spawn(_mp_worker, world, str(tmp_path / "ckpt.pt"), items=1, timeout=600)
    torch.cuda.set_device(0)
    plain, plain_beta = _trained(False)
    # Ranger / RAdam at lr 1e-5: a reordered gradient sum moves a weight by at most a few steps of 1e-5
    _near(ckpt, _full_state(plain, plain_beta), atol=1e-4)
    want = _run(plain, 6)
    for a, b in zip(losses, want):
        assert (a is None) == (b is None)
        if a is not None:
            for k in b:
                assert a[k] == pytest.approx(b[k], rel=1e-3, abs=1e-5), k
    _near(resumed, _full_state(plain, plain_beta), atol=2e-4)
