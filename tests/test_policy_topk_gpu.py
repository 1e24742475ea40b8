"""DiscreteActor.topk / recnn_discrete_topk / the sharded pair on the GPU, against the float64 restatement in
tests/_policy_topk_oracle.py, against the dense forward, and across chunkings, exclusions, ties and virtual ranks (the
pattern of test_reinforce_vocab_parallel_gpu.py: W shards in one process, the all-gather stood in for by concatenating
the records in rank order)."""
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
from recnn_b200.nn.arena import param_arena
from oracle import reinforce_oracle as RO
from tests import _policy_topk_oracle as TK
from tests._discrete import make_policy
from tests.test_reinforce_chunked_gpu import REORDER_BAR
from tests.test_reinforce_vocab_parallel_gpu import Virtual

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
L = _lib.lib()
# (S, H, items, rows): S % 4 == 0 (state read in place) and != 0 (re-pitched); rows below and above one CTA per row
SHAPES = [(52, 64, 1003, 40), (37, 32, 2000, 300), (20, 48, 5000, 9)]
KS = (1, 10, 16, 17, 64)
# fp32 error of a logit (3xTF32 GEMM or exact fp32, |z| <= ~15 here) and of a probability, relative to float64
Z_BAR = 2e-5
P_BAR = 5e-5


def _t(x):
    return torch.from_numpy(np.ascontiguousarray(x)).to(DEV)


def make_case(S, H, I, N, seed, spread=6.0):
    rng = np.random.default_rng(seed)
    p = RO.make_discrete_actor(rng, S, I, H)
    p["w2"] = (p["w2"] * spread).astype(np.float32)
    state = rng.normal(0, 1, (N, S)).astype(np.float32)
    return p, state


def call_topk(m, state, k, chunk=None, exclude=None):
    """(values, ids, error bits) of one explicit recnn_discrete_topk call."""
    d = m.dims
    n = state.shape[0]
    chunk = d.num_items if chunk is None or chunk >= d.num_items else chunk
    nbytes = L.recnn_discrete_topk_workspace_bytes(d, n, k, chunk)
    assert nbytes > 0
    ws = torch.empty(nbytes, dtype=torch.uint8, device=DEV)
    values = torch.empty(n, k, device=DEV)
    ids = torch.empty(n, k, dtype=torch.int64, device=DEV)
    flag = torch.full((1,), 7, dtype=torch.int32, device=DEV)
    n_ex = 0 if exclude is None else exclude.shape[1]
    _lib.check(L.recnn_discrete_topk(d, param_arena(m).data_ptr(), state.data_ptr(), n, k, _lib.ptr(exclude), n_ex,
                                     chunk, values.data_ptr(), ids.data_ptr(), flag.data_ptr(), ws.data_ptr(), nbytes,
                                     _lib.stream_ptr()))
    torch.cuda.synchronize()
    return values, ids, int(flag)


def check_against_oracle(values, ids, z, k, exclude=None, what="", min_sure=0.8):
    """ids equal the float64 ranking on every row whose k-th / (k+1)-th gap exceeds Z_BAR, in an order the float64
    logits confirm within Z_BAR; values within P_BAR of float64.  Returns (worst probability error, rows checked)."""
    want_v, want_i = TK.topk(z, k, None if exclude is None else exclude)
    got_v, got_i = values.cpu().numpy().astype(np.float64), ids.cpu().numpy()
    bar = Z_BAR * (1 + np.abs(z).max())
    sure = TK.boundary_gap(z, k, exclude) > bar
    assert sure.mean() >= min_sure, (what, sure.mean())
    for r in np.nonzero(sure)[0]:
        assert sorted(got_i[r]) == sorted(want_i[r]), (what, r, got_i[r], want_i[r])
    live = got_i >= 0
    zz = np.where(live, np.take_along_axis(z, np.maximum(got_i, 0), 1), -np.inf)
    assert (zz[:, 1:] <= zz[:, :-1] + bar).all(), what
    assert (np.diff(got_v, axis=1) <= 0).all(), what
    # values of the returned ids against float64 pi of the same ids
    M = z.max(1, keepdims=True)
    pi = np.exp(z - M) / np.exp(z - M).sum(1, keepdims=True)
    want_at = np.where(live, np.take_along_axis(pi, np.maximum(got_i, 0), 1), 0.0)
    err = np.abs(got_v - want_at) / np.maximum(want_v[:, :1], 1e-30)
    assert err.max() <= P_BAR, (what, err.max())
    assert ((got_i == -1) == (want_i == -1)).all(), what
    return float(err.max()), int(sure.sum())


def run_sweep():
    """Every shape x k x chunking against float64; chunked against one chunk."""
    worst = 0.0
    for S, H, I, N in SHAPES:
        p, state = make_case(S, H, I, N, S + I)
        m = make_policy(p, S, H, I)
        st = _t(state)
        z = TK.logits(p, state)
        bar = Z_BAR * (1 + np.abs(z).max())
        for k in KS:
            one_v, one_i, flag = call_topk(m, st, k)
            assert flag == 0
            worst = max(worst, check_against_oracle(one_v, one_i, z, k, what=(S, I, k, "one"))[0])
            for chunk in (128, 256):
                v, i, flag = call_topk(m, st, k, chunk)
                assert flag == 0
                worst = max(worst, check_against_oracle(v, i, z, k, what=(S, I, k, chunk))[0])
                sure = torch.from_numpy(TK.boundary_gap(z, k) > bar).to(DEV)
                assert torch.equal(i[sure].sort(1)[0], one_i[sure].sort(1)[0]), (S, I, k, chunk)
                same = (i == one_i).all(1)
                assert bool(same.any())
                r = float(((v - one_v).abs()[same] / one_v[same][:, :1]).max())
                assert r <= REORDER_BAR, (S, I, k, chunk, r)
                v2, i2, _ = call_topk(m, st, k, chunk)
                assert torch.equal(v2, v) and torch.equal(i2, i)
        print("topk S %d I %d N %d: ok" % (S, I, N))
    print("worst probability error %.2e" % worst)


def test_against_float64_and_across_chunkings():
    run_sweep()


def test_against_float64_on_the_cuda_core_back_end():
    """The same sweep with every GEMM on the exact-fp32 CUDA-core kernel, in a process of its own (the back end is
    fixed per process)."""
    code = "import sys; sys.path.insert(0, %r); from tests import test_policy_topk_gpu as T; T.run_sweep()" % ROOT
    env = dict(os.environ, RECNN_B200_MATH="simt")
    r = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, cwd=ROOT)
    print(r.stdout[-3000:], r.stderr[-3000:])
    assert r.returncode == 0


@pytest.mark.parametrize("S,H,I,N", SHAPES)
def test_single_chunk_values_are_the_forward_bits(S, H, I, N):
    p, state = make_case(S, H, I, N, 2 * S)
    m = make_policy(p, S, H, I)
    st = _t(state)
    probs = m(st)
    for k in (1, 17, 64):
        v, i, _ = call_topk(m, st, k)
        assert torch.equal(v, probs.gather(1, i)), k
        rest = probs.clone()
        rest.scatter_(1, i, -1.0)
        assert bool((v[:, -1] >= rest.max(1)[0]).all()), k
        pv, pi = m.topk(st, k)
        assert torch.equal(pv, v) and torch.equal(pi, i)


def _tie_policy(I, groups, S=36, H=32, seed=5):
    """A policy whose rows in each group of ids share one W2 row and bias (exact ties), above every other logit."""
    p, state = make_case(S, H, I, 24, seed, spread=1.0)
    for g, ids in enumerate(groups):
        p["w2"][ids] = p["w2"][ids[0]]
        p["b2"][ids] = 20.0 - 5 * g
    return p, state


def test_exact_ties_go_to_the_smaller_id():
    groups = [[500, 3, 128, 127, 129], [255, 256, 1002]]           # across the 128- and 256-chunk edges
    p, state = _tie_policy(1003, groups)
    m = make_policy(p, 36, 32, 1003)
    st = _t(state)
    want = torch.tensor(sorted(groups[0]) + sorted(groups[1]), device=DEV)
    for chunk in (None, 128, 256):
        v, i, _ = call_topk(m, st, 8, chunk)
        assert torch.equal(i, want.expand(24, 8)), (chunk, i[0])
        assert bool((v[:, :5] == v[:, :1]).all()) and bool((v[:, 5:] == v[:, 5:6]).all())


def test_exclusion():
    S, H, I, N = 37, 32, 2000, 40
    p, state = make_case(S, H, I, N, 11)
    m = make_policy(p, S, H, I)
    st = _t(state)
    z = TK.logits(p, state)
    rng = np.random.default_rng(3)
    ex = np.stack([rng.permutation(np.argsort(-z[r])[:80])[:60] for r in range(N)])     # mostly the best items
    ex[:, 50:] = -1                                                                       # padding
    ex[0, :] = -7
    for chunk in (None, 256):
        for k in (10, 64):
            v, i, flag = call_topk(m, st, k, chunk, _t(ex))
            assert flag == 0
            check_against_oracle(v, i, z, k, ex, what=("exclude", chunk, k))
            got = i.cpu().numpy()
            assert not any(np.isin(got[r], ex[r]).any() for r in range(N))
            if chunk is None:
                pv, pi = m.topk(st, k, exclude=_t(ex))
                assert torch.equal(pv, v) and torch.equal(pi, i)
    # an id >= num_items is refused; the C call reports it in bit 1
    bad = ex.copy()
    bad[5, 3] = I
    _, _, flag = call_topk(m, st, 10, None, _t(bad))
    assert flag == 1
    with pytest.raises(IndexError):
        m.topk(st, 10, exclude=_t(bad))


def test_fewer_eligible_items_than_k():
    S, H, I, N = 20, 16, 200, 6
    p, state = make_case(S, H, I, N, 4)
    m = make_policy(p, S, H, I)
    st = _t(state)
    ex = np.tile(np.arange(5, 200), (N, 1))[:, :195]              # items 0..4 left
    ex = np.concatenate([ex, np.full((N, 61), -1)], 1)            # E = 256 with padding
    v, i = m.topk(st, 12, exclude=_t(ex))
    z = TK.logits(p, state)
    want_v, want_i = TK.topk(z, 12, ex)
    assert (i[:, 5:] == -1).all() and (v[:, 5:] == 0).all()
    assert np.array_equal(np.sort(i[:, :5].cpu().numpy(), 1), np.tile(np.arange(5), (N, 1)))
    assert np.abs(v.cpu().numpy() - want_v).max() <= P_BAR * want_v.max()


def test_topk_leaves_the_policy_state_alone():
    S, H, I, N = 20, 16, 300, 8
    p, state = make_case(S, H, I, N, 8)
    m = make_policy(p, S, H, I)
    st = _t(state)
    m.select_action(st)
    saved = (len(m.saved_log_probs), len(m._saved), m._draws)
    arena = param_arena(m).clone()
    v, i = m.topk(st, 5)
    tgt = __import__("copy").deepcopy(m)
    tv, ti = tgt.topk(st, 5)
    assert (len(m.saved_log_probs), len(m._saved), m._draws) == saved
    assert torch.equal(param_arena(m), arena)
    assert torch.equal(tv, v) and torch.equal(ti, i)


# ----------------------------------------------------------------------------- 1M items
def test_million_items_memory_and_sampled_rows():
    """S 2570 / H 256, 2^20 items x 2,048 rows: the call's extra memory stays under 1.5 GB (the dense forward alone
    would hold 8.6 GB of probabilities) and sampled rows match a chunked float64 reference."""
    S, H, I, N, k = 2570, 256, 1 << 20, 2048, 64
    torch.manual_seed(0)
    m = recnn_b200.nn.DiscreteActor(S, I, H).to(DEV)
    with torch.no_grad():
        m.linear2.weight.mul_(8.0)
    flat = param_arena(m)
    st = torch.randn(N, S, device=DEV)
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    v, i = m.topk(st, k)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    print("1M items x %d rows: peak extra %.3f GB" % (N, peak / 1e9))
    assert peak < 1.5e9
    rows = torch.arange(0, N, N // 16, device=DEV)
    with torch.no_grad():
        x = st[rows].double()
        h = torch.relu(x @ m.linear1.weight.double().T + m.linear1.bias.double())
        z = torch.cat([h @ m.linear2.weight[c:c + 65536].double().T + m.linear2.bias[c:c + 65536].double()
                       for c in range(0, I, 65536)], 1).cpu().numpy()
    del flat
    check_against_oracle(v[rows], i[rows], z, k, what="1M", min_sure=0.7)


# ----------------------------------------------------------------------------- virtual ranks
def shard_topk(v, state, k, chunk=None, exclude=None, permute=None):
    """Both calls on every virtual rank: (per-rank values, per-rank ids, per-rank error bits)."""
    n = state.shape[0]
    st = _lib.stream_ptr()
    n_ex = 0 if exclude is None else exclude.shape[1]
    recs = []
    for r, m in enumerate(v.mods):
        d = m.dims
        c = d.num_items if chunk is None or chunk >= d.num_items else chunk
        nbytes = L.recnn_discrete_topk_workspace_bytes(d, n, k, c)
        ws = torch.empty(nbytes, dtype=torch.uint8, device=DEV)
        recs.append(torch.empty(L.recnn_vocab_topk_record_floats(n, k), device=DEV))
        _lib.check(L.recnn_discrete_shard_topk(d, v.vs(r), param_arena(m).data_ptr(), state.data_ptr(), n, k,
                                               _lib.ptr(exclude), n_ex, c, recs[r].data_ptr(), ws.data_ptr(), nbytes,
                                               st))
    gathered = torch.cat([recs[q] for q in (permute or range(v.world))])
    vals, ids, flags = [], [], []
    for r, m in enumerate(v.mods):
        vals.append(torch.empty(n, k, device=DEV))
        ids.append(torch.empty(n, k, dtype=torch.int64, device=DEV))
        flag = torch.full((1,), 9, dtype=torch.int32, device=DEV)
        _lib.check(L.recnn_discrete_shard_topk_finish(m.dims, v.vs(r), gathered.data_ptr(), n, k, _lib.ptr(exclude),
                                                      n_ex, vals[r].data_ptr(), ids[r].data_ptr(), flag.data_ptr(), st))
        flags.append(flag)
    torch.cuda.synchronize()
    return vals, ids, [int(f) for f in flags]


def _shard_tie_case(I, world, S=36, H=32, N=30):
    """Exact ties straddling every shard edge (lo - 1, lo, and the block's last item), above every other logit."""
    edges = sorted({e for lo, hi in TK.item_plan(I, world) for e in (lo - 1, lo, hi - 1) if 0 <= e < I})
    p, state = make_case(S, H, I, N, I + world, spread=2.0)
    p["w2"][edges] = p["w2"][edges[0]]
    p["b2"][edges] = 12.0
    return p, state, edges


@pytest.mark.parametrize("world", [1, 2, 3, 8])
def test_virtual_ranks(world):
    for S, H, I, N in [(52, 64, 1003, 40), (37, 32, 200, 17)]:      # 200 items over 8 ranks: 25 per block < k = 64
        p, state, edges = _shard_tie_case(I, world, S, H, N)
        v = Virtual(p, S, H, world)
        full = make_policy(p, S, H, I)
        st = _t(state)
        z = TK.logits(p, state)
        for k in (10, 64):
            for chunk in (None, 128):
                vals, ids, flags = shard_topk(v, st, k, chunk)
                assert flags == [0] * world
                for r in range(1, world):
                    assert torch.equal(vals[r], vals[0]) and torch.equal(ids[r], ids[0])
                check_against_oracle(vals[0], ids[0], z, k, what=("W", world, I, k, chunk), min_sure=0)
                want_i = TK.shard_topk(z, k, world)[1]
                top = min(len(edges), k)
                assert np.array_equal(ids[0][:, :top].cpu().numpy(), want_i[:, :top])
                assert np.array_equal(ids[0][:, :top].cpu().numpy(), np.tile(edges[:top], (N, 1)))
                if world == 1:
                    one_v, one_i, _ = call_topk(v.mods[0], st, k, chunk)
                    assert torch.equal(vals[0], one_v) and torch.equal(ids[0], one_i)
                if chunk is None:
                    blocks, _ = v.forward(st)
                    dense = torch.cat(blocks, 1)
                    assert torch.equal(vals[0], dense.gather(1, ids[0]))
        if world > 1:
            _, _, flags = shard_topk(v, st, 10, permute=[1, 0] + list(range(2, world)))
            assert all(f & 2 for f in flags), flags
        del full


def test_virtual_ranks_exclusion_on_shard_edges():
    S, H, I, N, world = 52, 64, 1003, 40, 3
    p, state, edges = _shard_tie_case(I, world, S, H, N)
    v = Virtual(p, S, H, world)
    st = _t(state)
    z = TK.logits(p, state)
    ex = np.full((N, 4), -1)
    ex[:, 0] = edges[1]
    ex[:, 1] = edges[-1]
    vals, ids, flags = shard_topk(v, st, 10, 128, _t(ex))
    assert flags == [0] * world
    want_v, want_i = TK.shard_topk(z, 10, world, ex)
    assert np.array_equal(ids[0][:, :len(edges) - 2].cpu().numpy(), want_i[:, :len(edges) - 2])
    check_against_oracle(vals[0], ids[0], z, 10, ex, what="W3 exclude", min_sure=0)
    ex[2, 3] = I
    _, _, flags = shard_topk(v, st, 10, 128, _t(ex))
    assert flags == [1] * world


# ----------------------------------------------------------------------------- the Python API at world 1
@pytest.fixture
def one_rank_group(tmp_path):
    import torch.distributed as dist
    torch.cuda.set_device(0)
    dist.init_process_group("nccl", init_method="file://" + str(tmp_path / "pg"), rank=0, world_size=1,
                            device_id=torch.device(DEV))
    yield
    dist.destroy_process_group()


def test_python_api_world1_equals_unsharded(one_rank_group, monkeypatch):
    S, H, I, N = 37, 32, 2000, 50
    torch.manual_seed(12)
    plain = recnn_b200.nn.DiscreteActor(S, I, H).to(DEV)
    shard = recnn_b200.nn.DiscreteActor(S, I, H).to(DEV)
    shard.load_state_dict(plain.state_dict())
    D.enable_vocab_parallel(shard)
    vp = shard.__dict__["_recnn_vp"]
    try:
        st = torch.randn(N, S, device=DEV)
        ex = torch.randint(-1, I, (N, 7), device=DEV)
        from recnn_b200.nn.update import reinforce as RF
        for chunk in (None, 256):
            if chunk is not None:
                monkeypatch.setattr(RF, "_chunk_items", lambda rows, items: min(chunk, items))
            for k, e in ((1, None), (17, ex), (64, ex)):
                a = plain.topk(st, k, exclude=e)
                b = shard.topk(st, k, exclude=e)
                assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1]), (chunk, k)
        with pytest.raises(IndexError):
            shard.topk(st, 3, exclude=torch.full((N, 1), I, device=DEV))
    finally:
        vp.comm.close()


# ----------------------------------------------------------------------------- W > 1 processes
def _topk_worker(rank, world, port, q):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    try:
        S, H, I, N = 52, 64, 1003, 48
        p, state = make_case(S, H, I, N, 77)
        m = make_policy(p, S, H, I).to(dev)
        D.enable_vocab_parallel(m)
        ex = torch.from_numpy(np.arange(N * 3).reshape(N, 3) % I).to(dev)
        v, i = m.topk(torch.from_numpy(state).to(dev), 16, exclude=ex)
        q.put((rank, v.cpu().numpy(), i.cpu().numpy()))
        torch.cuda.synchronize()
        m.__dict__["_recnn_vp"].comm.close()
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
    procs = [ctx.Process(target=_topk_worker, args=(r, world, port, q)) for r in range(world)]
    for pr in procs:
        pr.start()
    res = {r: (v, i) for r, v, i in (q.get(timeout=300) for _ in range(world))}
    for pr in procs:
        pr.join(timeout=60)
        assert pr.exitcode == 0
    S, H, I, N = 52, 64, 1003, 48
    p, state = make_case(S, H, I, N, 77)
    ex = np.arange(N * 3).reshape(N, 3) % I
    for r in range(world):
        assert np.array_equal(res[r][0].view(np.int32), res[0][0].view(np.int32))
        assert np.array_equal(res[r][1], res[0][1])
    check_against_oracle(torch.from_numpy(res[0][0]), torch.from_numpy(res[0][1]), TK.logits(p, state), 16, ex,
                         what=("processes", world))
