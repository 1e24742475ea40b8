"""The vocabulary-parallel REINFORCE policy on the GPU.

One GPU cannot run W > 1 ranks through the peer-memory protocol (every CTA of every rank must be resident at once; see
test_comm_world1_gpu.py), so the maths is checked with VIRTUAL ranks on one device: the C phases of W shards run in one
process, the all-gather is stood in for by concatenating the ranks' records in rank order (what recnn_comm_allgather
delivers) and the layer-1 all-reduce by an in-order fp32 sum (the order allreduce_kernel sums in).  The transport itself
is tested at world 1, and at W > 1 by the multi-process parametrisation, which needs W GPUs."""
from __future__ import annotations

import ctypes
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
from recnn_b200.utils.misc import DummyWriter
from oracle import reinforce_oracle as RO
from tests import _vocab_oracle as VO
from tests.test_comm_world1_gpu import World1Comm, _payload, CANARY
from tests.test_reinforce_chunked_gpu import REORDER_BAR, make_policy, policy_grad, unpack

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
L = _lib.lib()
# (S, H, items, rows, chunk): S % 4 == 0 (state read in place) and S % 4 != 0 (re-pitched image kept from the stats
# phase); local slices chunked with a ragged last chunk (W = 1, 3) and narrower than one chunk (W = 8)
SHAPES = [(52, 64, 1003, 40, 128), (37, 32, 2000, 33, 256)]


def _t(x, dtype=None):
    return torch.from_numpy(np.ascontiguousarray(x)).to(DEV) if dtype is None else torch.as_tensor(x, dtype=dtype,
                                                                                                     device=DEV)


class Virtual:
    """W shards of one DiscreteActor as W modules on one device."""

    def __init__(self, p, S, H, world):
        self.items = p["w2"].shape[0]
        self.world = world
        self.shards = RO.shard_policy(p, world)
        self.mods = [make_policy({"w1": p["w1"], "b1": p["b1"], "w2": sh["w2"], "b2": sh["b2"]}, S, H, len(sh["b2"]))
                     for sh in self.shards]

    def vs(self, r):
        return _lib.VocabShard(self.shards[r]["offset"], self.items, r, self.world)

    def grad(self, state, action, blp, ret, method, K, chunk, permute=None):
        """Both phases on every rank: (losses, flags [W, 2], per-rank gradient dicts with the all-reduced layer 1)."""
        n = state.shape[0]
        st = _lib.stream_ptr()
        recs, scratch, chunks = [], [], []
        for r, m in enumerate(self.mods):
            d = m.dims
            c = chunk if chunk < d.num_items else d.num_items
            chunks.append(c)
            scratch.append(torch.empty(L.recnn_reinforce_scratch_floats(d, n, c), device=DEV))
            recs.append(torch.empty(L.recnn_vocab_record_floats(n), device=DEV))
            _lib.check(L.recnn_reinforce_shard_stats(d, self.vs(r), param_arena(m).data_ptr(), state.data_ptr(),
                                                     action.data_ptr(), n, c, recs[r].data_ptr(),
                                                     scratch[r].data_ptr(), st))
        order = permute or list(range(self.world))
        gathered = torch.cat([recs[q] for q in order])
        grads, outs = [], []
        for r, m in enumerate(self.mods):
            g = torch.full_like(param_arena(m), float("nan"))
            out = torch.zeros(3, device=DEV)
            _lib.check(L.recnn_reinforce_shard_grad(m.dims, self.vs(r), param_arena(m).data_ptr(), g.data_ptr(),
                                                    state.data_ptr(), action.data_ptr(), _lib.ptr(blp), ret.data_ptr(),
                                                    n, method, K, chunks[r], gathered.data_ptr(), out.data_ptr(),
                                                    scratch[r].data_ptr(), st))
            grads.append(g)
            outs.append(out)
        layer1 = D.layer1_floats(self.mods[0].dims)
        acc = grads[0][:layer1].clone()
        for g in grads[1:]:
            acc += g[:layer1]
        for g in grads:
            g[:layer1] = acc
        torch.cuda.synchronize()
        return ([float(o[0]) for o in outs], [o.view(torch.int32)[1:].tolist() for o in outs],
                [unpack(g, m) for g, m in zip(grads, self.mods)])

    def forward(self, state):
        """(column blocks, gathered records) of the sharded forward."""
        n = state.shape[0]
        st = _lib.stream_ptr()
        blocks, recs = [], []
        for r, m in enumerate(self.mods):
            d = m.dims
            blocks.append(torch.empty(n, d.num_items, device=DEV))
            recs.append(torch.empty(L.recnn_vocab_record_floats(n), device=DEV))
            scratch = torch.empty(L.recnn_discrete_scratch_floats(d, n, 0), device=DEV)
            _lib.check(L.recnn_discrete_shard_forward(d, self.vs(r), param_arena(m).data_ptr(), state.data_ptr(), n,
                                                      blocks[r].data_ptr(), recs[r].data_ptr(), scratch.data_ptr(), st))
        gathered = torch.cat(recs)
        flag = torch.zeros(1, dtype=torch.int32, device=DEV)
        for r, m in enumerate(self.mods):
            _lib.check(L.recnn_discrete_shard_finish(m.dims, self.vs(r), gathered.data_ptr(), n, blocks[r].data_ptr(),
                                                     flag.data_ptr(), st))
        assert int(flag) == 0
        return blocks, gathered

    def _pick(self, draws, n):
        action = torch.empty(n, dtype=torch.int64, device=DEV)
        logp = torch.empty(n, device=DEV)
        flag = torch.zeros(1, dtype=torch.int32, device=DEV)
        _lib.check(L.recnn_discrete_shard_pick(self.world, torch.cat(draws).data_ptr(), n, action.data_ptr(),
                                               logp.data_ptr(), flag.data_ptr(), _lib.stream_ptr()))
        return action, logp, int(flag)

    def sample(self, blocks, gathered, uniforms=None, seed=0, draw=1):
        n = blocks[0].shape[0]
        draws = []
        for r, m in enumerate(self.mods):
            draws.append(torch.empty(2 * n, device=DEV))
            _lib.check(L.recnn_discrete_shard_sample(m.dims, self.vs(r), gathered.data_ptr(), blocks[r].data_ptr(), n,
                                                     _lib.ptr(uniforms), seed, draw, draws[r].data_ptr(),
                                                     _lib.stream_ptr()))
        return self._pick(draws, n)

    def log_prob(self, blocks, action):
        n = blocks[0].shape[0]
        draws, oob = [], torch.zeros(1, dtype=torch.int32, device=DEV)
        for r, m in enumerate(self.mods):
            draws.append(torch.empty(2 * n, device=DEV))
            _lib.check(L.recnn_discrete_shard_log_prob(m.dims, self.vs(r), blocks[r].data_ptr(), n, action.data_ptr(),
                                                       draws[r].data_ptr(), oob.data_ptr(), _lib.stream_ptr()))
        a, lp, flag = self._pick(draws, n)
        return lp, flag, int(oob)


def _case(S, H, I, R, seed, world):
    rng = np.random.default_rng(seed)
    p = RO.make_discrete_actor(rng, S, I, H)
    state = rng.normal(0, 1, (R, S)).astype(np.float32)
    blp = np.log(rng.uniform(1e-4, 5e-4, R)).astype(np.float32)
    ret = rng.normal(0, 1, R).astype(np.float32)
    action = rng.integers(0, I, R)
    edges = sorted({e for sh in RO.shard_policy(p, world)
                    for e in (sh["offset"] - 1, sh["offset"], sh["offset"] + len(sh["b2"]) - 1) if 0 <= e < I})
    action[:len(edges)] = edges[:R]
    return p, state, action, blp, ret


def run_virtual_sweep():
    """Every shape x W x method: loss and gradients against the float64 oracle (the chunked-gradient tests' bar) and
    against the unsharded chunked CUDA call (reordering bar); the loss has the same bits on every rank."""
    for S, H, I, R, chunk in SHAPES:
        for world in (1, 2, 3, 8):
            p, state, action, blp, ret = _case(S, H, I, R, S + I + world, world)
            v = Virtual(p, S, H, world)
            full = make_policy(p, S, H, I)
            st, at, bt, rt = _t(state), _t(action), _t(blp), _t(ret)
            for method in (RO.BASIC, RO.CORRECTED, RO.TOPK):
                beta = None if method == RO.BASIC else bt
                losses, flags, grads = v.grad(st, at, beta, rt, method, 10, chunk)
                assert flags == [[0, 0]] * world, flags
                assert len({np.float32(x).tobytes() for x in losses}) == 1, losses
                want_loss, want, _ = RO.reinforce_policy_grad(p, state, action, None if beta is None else blp, ret,
                                                              method, 10)
                one_loss, _, one = policy_grad(full, st, at, beta, rt, method, 10, chunk)
                assert losses[0] == pytest.approx(want_loss, rel=2e-4, abs=1e-4 * (1 + abs(want_loss)))
                assert losses[0] == pytest.approx(one_loss, rel=1e-5, abs=1e-6)
                got = {"w1": grads[0]["w1"], "b1": grads[0]["b1"],
                       "w2": torch.cat([g["w2"] for g in grads]), "b2": torch.cat([g["b2"] for g in grads])}
                for k in got:
                    assert torch.isfinite(got[k]).all(), k
                    scale = np.abs(want[k]).max()
                    err = np.abs(got[k].cpu().numpy() - want[k]).max()
                    assert err <= 3e-4 * scale, (S, I, world, method, k, err, scale)
                    r = float((got[k] - one[k]).abs().max() / one[k].abs().max())
                    assert r <= REORDER_BAR, (S, I, world, method, k, r)
                for g in grads[1:]:
                    assert torch.equal(g["w1"], grads[0]["w1"]) and torch.equal(g["b1"], grads[0]["b1"])
            print("virtual ranks S %d I %d W %d: ok" % (S, I, world))


def test_virtual_ranks_against_the_oracle():
    run_virtual_sweep()


def test_virtual_ranks_on_the_cuda_core_back_end():
    """The same sweep with every GEMM on the exact-fp32 CUDA-core kernel, in a process of its own (the back end is fixed
    per process)."""
    code = "import sys; sys.path.insert(0, %r); from tests import test_reinforce_vocab_parallel_gpu as T; " \
           "T.run_virtual_sweep()" % ROOT
    env = dict(os.environ, RECNN_B200_MATH="simt")
    r = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, cwd=ROOT)
    print(r.stdout[-3000:], r.stderr[-3000:])
    assert r.returncode == 0


@pytest.mark.parametrize("S,H,I,R,chunk", SHAPES)
def test_world1_is_bit_identical_to_the_chunked_call(S, H, I, R, chunk):
    p, state, action, blp, ret = _case(S, H, I, R, 3 * S, 1)
    v = Virtual(p, S, H, 1)
    st, at, bt, rt = _t(state), _t(action), _t(blp), _t(ret)
    for method in (RO.BASIC, RO.TOPK):
        beta = None if method == RO.BASIC else bt
        losses, flags, grads = v.grad(st, at, beta, rt, method, 10, chunk)
        loss, _, want = policy_grad(v.mods[0], st, at, beta, rt, method, 10, chunk)
        assert np.float32(losses[0]).tobytes() == np.float32(loss).tobytes()
        for k in want:
            assert torch.equal(grads[0][k], want[k]), k


def test_gathered_records_out_of_rank_order_are_flagged():
    p, state, action, blp, ret = _case(52, 64, 1003, 40, 5, 3)
    v = Virtual(p, 52, 64, 3)
    _, flags, _ = v.grad(_t(state), _t(action), None, _t(ret), RO.BASIC, 1, 128, permute=[1, 0, 2])
    assert all(f[1] == 1 for f in flags), flags


# ----------------------------------------------------------------------------- forward and draws
def _forward_case(world, n=300, S=52, H=64, I=1003, seed=0):
    rng = np.random.default_rng(seed + world)
    p = RO.make_discrete_actor(rng, S, I, H)
    p["w2"] = (p["w2"] * 6).astype(np.float32)
    state = rng.normal(0, 1, (n, S)).astype(np.float32)
    return p, state, Virtual(p, S, H, world), make_policy(p, S, H, I)


@pytest.mark.parametrize("world", [2, 3, 8])
def test_forward_blocks_and_replayed_draws(world):
    p, state, v, full = _forward_case(world)
    st = _t(state)
    blocks, gathered = v.forward(st)
    probs = torch.cat(blocks, 1)
    want = full(st)
    assert float((probs - want).abs().max()) <= 1e-6 * float(want.abs().max())
    assert float((probs.double().sum(1) - 1).abs().max()) <= 1e-5
    u = np.random.default_rng(world).random(state.shape[0]).astype(np.float32)
    a, lp, flag = v.sample(blocks, gathered, uniforms=_t(u))
    assert flag == 0
    full.uniform_source = lambda n: u
    ref_a, ref_lp = full._sample(want)
    _, _, margin = RO.categorical_sample(want.double().cpu().numpy(), u)
    keep = torch.from_numpy(margin > 1e-5).to(DEV)
    assert int(keep.sum()) > 0.9 * state.shape[0]
    assert torch.equal(a[keep], ref_a[keep])
    assert float((lp[keep] - ref_lp[keep]).abs().max()) <= 1e-5
    # the log-prob of given ids at every shard edge
    edges = sorted({e for sh in v.shards for e in (sh["offset"] - 1, sh["offset"], sh["offset"] + len(sh["b2"]) - 1)
                    if 0 <= e < 1003})
    ids = np.random.default_rng(1).integers(0, 1003, state.shape[0])
    ids[:len(edges)] = edges
    lp2, flag2, oob = v.log_prob(blocks, _t(ids))
    assert flag2 == 0 and oob == 0
    want_lp = RO.categorical_log_prob(want.double().cpu().numpy(), ids)
    assert np.abs(lp2.cpu().numpy() - want_lp).max() <= 1e-5
    ids[3] = 1003
    _, flag3, oob3 = v.log_prob(blocks, _t(ids))
    assert oob3 == 1 and flag3 == 1


def test_world1_forward_and_draws_are_bit_identical():
    p, state, v, full = _forward_case(1)
    st = _t(state)
    blocks, gathered = v.forward(st)
    want = full(st)
    assert torch.equal(blocks[0], want)
    u = _t(np.random.default_rng(2).random(state.shape[0]).astype(np.float32))
    for uniforms in (u, None):
        a, lp, flag = v.sample(blocks, gathered, uniforms=uniforms, seed=1234, draw=5)
        ra = torch.empty_like(a)
        rl = torch.empty_like(lp)
        _lib.check(L.recnn_categorical_sample(want.data_ptr(), want.shape[0], want.shape[1], want.stride(0),
                                              _lib.ptr(uniforms), 1234, 5, ra.data_ptr(), rl.data_ptr(),
                                              _lib.stream_ptr()))
        assert flag == 0
        assert torch.equal(a, ra) and torch.equal(lp, rl)


def test_philox_draws_follow_the_softmax_at_w3():
    """One state repeated over 60,000 rows, 13 items over 3 ranks (5, 5, 3): the seeded Philox draws pass a
    chi-square test against the softmax."""
    from scipy.stats import chisquare
    p, _, v, full = _forward_case(3, S=8, H=16, I=13, seed=40)
    rng = np.random.default_rng(9)
    state = np.repeat(rng.normal(0, 1, (1, 8)).astype(np.float32), 60_000, 0)
    blocks, gathered = v.forward(_t(state))
    a, _, flag = v.sample(blocks, gathered, seed=777, draw=3)
    assert flag == 0
    counts = np.bincount(a.cpu().numpy(), minlength=13)
    probs = full(_t(state[:1])).double().cpu().numpy()[0]
    probs /= probs.sum()
    assert probs.min() * 60_000 > 50
    res = chisquare(counts, probs * counts.sum())
    print("chi-square %.2f, p %.3f" % (res.statistic, res.pvalue))
    assert res.pvalue > 1e-3


# ----------------------------------------------------------------------------- the all-gather at world 1
def test_allgather_moves_every_bit_pattern_and_interleaves_with_allreduce():
    """World 1: the all-gather copies every fp32 / int32 bit pattern (NaN payloads, ids) unchanged at sizes 1..4097 and
    the capacity, back to back (both epoch parities) and interleaved with recnn_comm_allreduce on the same
    communicator; one float over the capacity is refused before any launch."""
    comm = World1Comm(4099)
    rng = np.random.default_rng(31)
    st = torch.cuda.current_stream().cuda_stream
    try:
        for i, n in enumerate((1, 2, 3, 7, 1001, 4096, 4097, comm.capacity)):
            for _ in range(2):
                x = _payload(n, rng) if i % 2 else torch.from_numpy(rng.integers(-1, 10**6, n).astype(np.int32)).to(DEV)
                out = torch.full((n + 64,), CANARY, dtype=torch.int32, device=DEV)
                _lib.check(L.recnn_comm_allgather(comm.handle, x.data_ptr(), n, out.data_ptr(), st))
                y = torch.randn(n + (n % 2), device=DEV)
                y0 = y.clone()
                comm.all_reduce(y)
                torch.cuda.synchronize()
                assert torch.equal(out[:n].cpu(), x.cpu()), n
                assert bool((out[n:] == CANARY).all())
                assert torch.equal(y.view(torch.int32), y0.view(torch.int32))
        k0 = L.recnn_b200_launch_count()
        big = torch.zeros(comm.capacity + 1, device=DEV)
        with pytest.raises(_lib.RecnnError, match="capacity"):
            _lib.check(L.recnn_comm_allgather(comm.handle, big.data_ptr(), big.numel(), big.data_ptr(), st))
        assert L.recnn_b200_launch_count() == k0
    finally:
        comm.close()


# ----------------------------------------------------------------------------- the Python API at world 1
@pytest.fixture
def one_rank_group(tmp_path):
    import torch.distributed as dist
    torch.cuda.set_device(0)
    dist.init_process_group("nccl", init_method="file://" + str(tmp_path / "pg"), rank=0, world_size=1,
                            device_id=torch.device(DEV))
    yield
    dist.destroy_process_group()


def _policy_pair(S, H, I, seed):
    torch.manual_seed(seed)
    a = recnn_b200.nn.DiscreteActor(S, I, H).to(DEV)
    b = recnn_b200.nn.DiscreteActor(S, I, H).to(DEV)
    b.load_state_dict(a.state_dict())
    D.enable_vocab_parallel(b)
    return a, b


def _bits(t):
    return t.detach().contiguous().view(torch.int32).cpu()


@pytest.mark.parametrize("variant", ["basic_adam", "topk_torch_sgd"])
def test_python_api_world1_equals_unsharded(one_rank_group, variant):
    S, H, I, N, T = 52, 64, 1003, 16, 3
    plain, shard = _policy_pair(S, H, I, 21)
    vp = shard.__dict__["_recnn_vp"]
    assert (vp.lo, vp.hi, vp.num_items, vp.world) == (0, I, I, 1)
    if variant == "basic_adam":
        method = recnn_b200.nn.ChooseREINFORCE.basic_reinforce
        opts = [recnn_b200.optim.Adam(m.parameters(), lr=1e-3) for m in (plain, shard)]
    else:
        method = recnn_b200.nn.ChooseREINFORCE.reinforce_with_TopK_correction
        opts = [torch.optim.SGD(m.parameters(), lr=1e-2) for m in (plain, shard)]
    rng = np.random.default_rng(5)
    bw = torch.from_numpy(rng.normal(0, 0.3, (I, S)).astype(np.float32)).to(DEV)
    beta = lambda s, action=None: torch.softmax(s @ bw.T, dim=1)       # noqa: E731
    for update in range(3):
        for t in range(T):
            state = torch.from_numpy(rng.normal(0, 1, (N, S)).astype(np.float32)).to(DEV)
            outs = []
            for m in (plain, shard):
                if variant == "basic_adam":
                    outs.append(m.select_action(state))
                else:
                    outs.append(m._select_action_with_TopK_correction(state, beta, None, K=10, writer=DummyWriter(),
                                                                      step=t))
                m.rewards.append(torch.tensor(float(t + update)))
            assert torch.equal(outs[0], outs[1])
            for k in ("saved_log_probs", "correction", "lambda_k"):
                for x, y in zip(getattr(plain, k), getattr(shard, k)):
                    assert torch.equal(x, y), k
        losses = [recnn_b200.nn.ChooseREINFORCE(method)(m, o) for m, o in zip((plain, shard), opts)]
        assert _bits(losses[0]).tolist() == _bits(losses[1]).tolist()
        assert torch.equal(_bits(param_arena(plain)), _bits(param_arena(shard))), update
        assert torch.equal(_bits(grad_arena(plain)), _bits(grad_arena(shard))), update
    # error paths on the sharded policy
    shard._saved.append({"state": state, "action": torch.full((N,), I, dtype=torch.int64, device=DEV),
                         "beta_log_prob": None})
    shard.rewards.append(torch.tensor(1.0))
    with pytest.raises(IndexError):
        recnn_b200.nn.ChooseREINFORCE()(shard, opts[1])
    with pytest.raises(IndexError):
        shard._shard_log_prob(shard(state), torch.full((N,), -1, dtype=torch.int64))
    with pytest.raises(RuntimeError, match="ChooseREINFORCE"):
        recnn_b200.nn.reinforce_update({"state": state, "action": torch.zeros(N, I)}, {}, {"policy_net": shard}, {})
    vp.comm.close()


# ----------------------------------------------------------------------------- one rank's share of config 5
def test_config5_rank_share_memory_is_bounded():
    """S 2570 / H 256, 1M items over 8 ranks (125,000 local) x 163,840 saved rows: the stats and gradient phases of one
    virtual rank, with every other rank's record standing in as a copy of this one's.  The call's extra memory is the
    scratch (one logits chunk, the state image, two hidden buffers, the partials) plus the records."""
    from recnn_b200.nn.update import reinforce as RF
    S, H, I, world, R = 2570, 256, 1_000_000, 8, 163_840
    lo, hi = D.vocab_shard(I, 7, world)
    torch.manual_seed(3)
    with torch.device(DEV):
        m = recnn_b200.nn.DiscreteActor(S, hi - lo, H)
        state = torch.randn(R, S)
        action = torch.randint(lo, hi, (R,))
        ret = torch.randn(R)
    d = m.dims
    chunk = RF._chunk_items(R, d.num_items)
    g = grad_arena(m)
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    scratch = torch.empty(L.recnn_reinforce_scratch_floats(d, R, chunk), device=DEV)
    rec = torch.empty(L.recnn_vocab_record_floats(R), device=DEV)
    vs = _lib.VocabShard(lo, I, 7, world)
    _lib.check(L.recnn_reinforce_shard_stats(d, vs, param_arena(m).data_ptr(), state.data_ptr(), action.data_ptr(), R,
                                             chunk, rec.data_ptr(), scratch.data_ptr(), _lib.stream_ptr()))
    gathered = rec.repeat(world)
    hdr = gathered.view(world, -1)[:, :4].view(torch.int32)
    for q in range(world):
        hdr[q, :2] = torch.tensor(D.vocab_shard(I, q, world), dtype=torch.int32)
    out = torch.zeros(3, device=DEV)
    _lib.check(L.recnn_reinforce_shard_grad(d, vs, param_arena(m).data_ptr(), g.data_ptr(), state.data_ptr(),
                                            action.data_ptr(), None, ret.data_ptr(), R, RO.BASIC, 1, chunk,
                                            gathered.data_ptr(), out.data_ptr(), scratch.data_ptr(), _lib.stream_ptr()))
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    print("config-5 rank share: chunk %d, scratch %.2f GB, peak extra %.2f GB"
          % (chunk, scratch.numel() * 4 / 1e9, peak / 1e9))
    assert out.view(torch.int32)[1:].tolist() == [0, 0]
    assert np.isfinite(float(out[0]))
    assert peak <= scratch.numel() * 4 + (world + 1) * rec.numel() * 4 + (64 << 20)
    assert peak < 6e9


# ----------------------------------------------------------------------------- W > 1 processes
def _vp_worker(rank, world, port, q):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    try:
        S, H, I, R = 52, 64, 1003, 48
        p, state, action, blp, ret = _case(S, H, I, R, 77, world)
        m = recnn_b200.nn.DiscreteActor(S, I, H)
        if rank == 0:
            with torch.no_grad():
                for name, k in (("linear1.weight", "w1"), ("linear1.bias", "b1"), ("linear2.weight", "w2"),
                                ("linear2.bias", "b2")):
                    m.get_parameter(name).copy_(torch.from_numpy(p[k]))
        m = m.to(dev)
        D.enable_vocab_parallel(m)
        opt = recnn_b200.optim.SGD(m.parameters(), lr=0.1)
        for t in range(2):
            rows = slice(t * R // 2, (t + 1) * R // 2)
            m._saved.append({"state": torch.from_numpy(state[rows]).to(dev), "action": torch.from_numpy(action[rows]).to(dev),
                             "beta_log_prob": torch.from_numpy(blp[rows]).to(dev), "K": 10})
            m.rewards.append(torch.tensor(float(t)))
        loss = recnn_b200.nn.ChooseREINFORCE(recnn_b200.nn.ChooseREINFORCE.reinforce_with_TopK_correction)(m, opt)
        vp = m.__dict__["_recnn_vp"]
        q.put((rank, {"loss": float(loss), "lo": vp.lo, "hi": vp.hi,
                      "w1": m.linear1.weight.detach().cpu().numpy(), "b1": m.linear1.bias.detach().cpu().numpy(),
                      "gw1": m.linear1.weight.grad.cpu().numpy(), "gw2": m.linear2.weight.grad.cpu().numpy(),
                      "gb2": m.linear2.bias.grad.cpu().numpy()}))
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
    procs = [ctx.Process(target=_vp_worker, args=(r, world, port, q)) for r in range(world)]
    for pr in procs:
        pr.start()
    res = dict(q.get(timeout=300) for _ in range(world))
    for pr in procs:
        pr.join(timeout=60)
        assert pr.exitcode == 0
    S, H, I, R = 52, 64, 1003, 48
    p, state, action, blp, ret = _case(S, H, I, R, 77, world)
    full = make_policy(p, S, H, I)
    full._saved = [{"state": _t(state[:R // 2]), "action": _t(action[:R // 2]), "beta_log_prob": _t(blp[:R // 2]),
                    "K": 10},
                   {"state": _t(state[R // 2:]), "action": _t(action[R // 2:]), "beta_log_prob": _t(blp[R // 2:]),
                    "K": 10}]
    full.rewards = [torch.tensor(0.0), torch.tensor(1.0)]
    want_loss = recnn_b200.nn.ChooseREINFORCE(recnn_b200.nn.ChooseREINFORCE.reinforce_with_TopK_correction)(full, None,
                                                                                                         learn=False)
    gw2 = torch.cat([torch.from_numpy(res[r]["gw2"]) for r in range(world)])
    gb2 = torch.cat([torch.from_numpy(res[r]["gb2"]) for r in range(world)])
    for r in range(world):
        assert res[r]["loss"] == res[0]["loss"]
        assert np.array_equal(res[r]["w1"].view(np.int32), res[0]["w1"].view(np.int32))
        assert np.array_equal(res[r]["b1"].view(np.int32), res[0]["b1"].view(np.int32))
        assert np.array_equal(res[r]["gw1"].view(np.int32), res[0]["gw1"].view(np.int32))
    assert res[0]["loss"] == pytest.approx(float(want_loss), rel=1e-5, abs=1e-6)
    for got, want in ((gw2, full.linear2.weight.grad), (gb2, full.linear2.bias.grad),
                      (torch.from_numpy(res[0]["gw1"]), full.linear1.weight.grad)):
        r = float((got - want.cpu()).abs().max() / want.abs().max())
        assert r <= REORDER_BAR, r
