"""The workspace contract of the serving, ranking, log-prob and sharded entry points, extended to every caller buffer.

test_workspace_bounds_gpu.py holds the training step and forward calls to their queried sizes.  Here the same two
checks (check_exact_size's canary and bit comparison, check_too_small's refusal) cover the calls that serve, rank and
score items, and every caller buffer of theirs that has a size contract gets a window of its own: the byte workspace,
each record (sized by its *_record_floats query; at world 1 the gathered buffer a finish phase reads is a second window
the record is copied into), and each output ([n, k] ids / values, ranks, log-probs, probabilities, slate reductions).
A window sits at exactly its size, 16 bytes into its own buffer with GUARD canary bytes behind it.  For each call:
  - every window's canaries survive on both sides;
  - the outputs, the records and the state the calls write are the bits of a run on generous zero-filled buffers, so a
    read past a window (canary there, zeros in the generous run) shows up too;
  - one byte less of workspace is refused with RECNN_E_WORKSPACE before anything runs: the launch count does not move,
    the error flags keep the sentinel written before the call and no window is touched.
Every write stays inside a live allocation: an overrun changes a canary, it never faults.

COVERED lists every entry point of include/recnn_b200.h that takes a caller workspace or writes a gathered record, with
the test that bounds it; test_workspace_bounds_host.py fails when a declaration is missing from it."""
from __future__ import annotations

import numpy as np
import pytest
import torch

import recnn_b200
from recnn_b200 import _lib
from recnn_b200.nn.arena import grad_arena, param_arena
from tests.test_workspace_bounds_gpu import (CANARY, DEV, DISCRETE, E_WORKSPACE, GUARD, L, OFFSET, _bytes, _critic_rank,
                                             _discrete, check_too_small)

pytestmark = pytest.mark.gpu

# entry point -> the test that holds it to its sizes ("file::test" when another file does)
COVERED = {
    "recnn_step_workspace_bytes": "test_workspace_bounds_gpu.py::test_step",
    "recnn_ddpg_step": "test_workspace_bounds_gpu.py::test_step",
    "recnn_td3_step": "test_workspace_bounds_gpu.py::test_step",
    "recnn_retrieve_workspace_bytes": "test_retrieval_topk_sets",
    "recnn_retrieve_topk": "test_workspace_bounds_gpu.py::test_retrieval",
    "recnn_retrieve_topk_sets": "test_retrieval_topk_sets",
    "recnn_retrieve_rank_workspace_bytes": "test_retrieval_rank",
    "recnn_retrieve_rank": "test_retrieval_rank",
    "recnn_retrieve_rank_sets": "test_retrieval_rank",
    "recnn_slate_distances": "test_slate_distances",
    "recnn_critic_serve_workspace_bytes": "test_critic_serving",
    "recnn_critic_topk": "test_critic_serving",
    "recnn_critic_rank": "test_critic_serving",
    "recnn_discrete_topk_workspace_bytes": "test_policy_topk_and_slates",
    "recnn_discrete_topk": "test_policy_topk_and_slates",
    "recnn_discrete_topk_sets": "test_policy_topk_and_slates",
    "recnn_discrete_sample_topk": "test_policy_topk_and_slates",
    "recnn_discrete_sample_topk_sets": "test_policy_topk_and_slates",
    "recnn_vocab_topk_record_floats": "test_sharded_topk_and_slates",
    "recnn_vocab_sample_topk_record_floats": "test_sharded_topk_and_slates",
    "recnn_discrete_shard_topk": "test_sharded_topk_and_slates",
    "recnn_discrete_shard_topk_sets": "test_sharded_topk_and_slates",
    "recnn_discrete_shard_topk_finish": "test_sharded_topk_and_slates",
    "recnn_discrete_shard_sample_topk": "test_sharded_topk_and_slates",
    "recnn_discrete_shard_sample_topk_sets": "test_sharded_topk_and_slates",
    "recnn_discrete_shard_sample_topk_finish": "test_sharded_topk_and_slates",
    "recnn_discrete_rank_workspace_bytes": "test_policy_rank_and_log_prob",
    "recnn_discrete_rank": "test_policy_rank_and_log_prob",
    "recnn_discrete_rank_sets": "test_policy_rank_and_log_prob",
    "recnn_discrete_log_prob": "test_policy_rank_and_log_prob",
    "recnn_vocab_record_floats": "test_sharded_rank_and_log_prob",
    "recnn_vocab_rank_record_floats": "test_sharded_rank_and_log_prob",
    "recnn_discrete_shard_rank_stats": "test_sharded_rank_and_log_prob",
    "recnn_discrete_shard_rank": "test_sharded_rank_and_log_prob",
    "recnn_discrete_shard_rank_sets": "test_sharded_rank_and_log_prob",
    "recnn_discrete_shard_rank_finish": "test_sharded_rank_and_log_prob",
    "recnn_vocab_log_prob_finish": "test_sharded_rank_and_log_prob",
    "recnn_reinforce_shard_stats": "test_sharded_rank_and_log_prob",
    "recnn_beta_workspace_bytes": "test_beta_shard_phases",
    "recnn_beta_step": "test_workspace_bounds_gpu.py::test_beta_step",
    "recnn_beta_shard_begin": "test_beta_shard_phases",
    "recnn_beta_shard_rows": "test_beta_shard_phases",
    "recnn_beta_shard_end": "test_beta_shard_phases",
    "recnn_beta_log_prob_workspace_bytes": "test_beta_log_prob",
    "recnn_beta_log_prob": "test_beta_log_prob",
    "recnn_beta_shard_log_prob_stats": "test_beta_log_prob",
    "recnn_discrete_value_workspace_bytes": "test_workspace_bounds_gpu.py::test_item_id_critic_step",
    "recnn_discrete_value_step": "test_workspace_bounds_gpu.py::test_item_id_critic_step",
    "recnn_discrete_value_shard_begin": "test_workspace_bounds_gpu.py::test_item_id_critic_shard_phases",
    "recnn_discrete_value_shard_merge": "test_workspace_bounds_gpu.py::test_item_id_critic_shard_phases",
    "recnn_discrete_value_shard_end": "test_workspace_bounds_gpu.py::test_item_id_critic_shard_phases",
    "recnn_discrete_value_dp_grad_floats": "test_item_id_critic_data_parallel",
    "recnn_discrete_value_dp_record_floats": "test_item_id_critic_data_parallel",
    "recnn_discrete_value_dp_workspace_bytes": "test_item_id_critic_data_parallel",
    "recnn_discrete_value_dp_begin": "test_item_id_critic_data_parallel",
    "recnn_discrete_value_dp_end": "test_item_id_critic_data_parallel",
}

SENTINEL = 0x5EED5EED       # written to every error flag before a refused call: it must still be there after
KS = [1, 17, 64]            # 17 crosses the 16 -> 64 register-list template
STAGE = 4096                # kSetStage: longer sets are searched in global memory


# ---------------------------------------------------------------- the windows
def _lay(sizes, canary):
    """name -> (buffer, window): the window is sizes[name] bytes, 16 bytes into a buffer of canary with GUARD bytes of
    it behind (canary False: the generous run, the window at the start of a zero-filled buffer GUARD bytes longer)"""
    out = {}
    for name, n in sizes.items():
        if canary:
            buf = torch.full((OFFSET + n + GUARD,), CANARY, dtype=torch.uint8, device=DEV)
            out[name] = (buf, buf[OFFSET:OFFSET + n])
        else:
            buf = torch.zeros(n + GUARD, dtype=torch.uint8, device=DEV)
            out[name] = (buf, buf[:n])
    return out


def _gather(src, dst):
    """the all-gather of one rank's record at world 1: a copy, on the stream the calls run on"""
    def run(w, nbytes):
        w[dst].copy_(w[src])
        return 0
    return False, run


class _At:
    """a window given as an address (check_too_small owns the short workspace)"""

    def __init__(self, p):
        self.p = p

    def data_ptr(self):
        return self.p


def check_windows(sizes, calls, state=(), flags=(), partial=()):
    """sizes: name -> bytes of every caller buffer with a size contract, "ws" being the byte workspace when there is
    one.  calls: [(takes_ws, run(win, ws_bytes) -> status)] in order; win maps a name to its window (a uint8 tensor).
    state: the other device tensors the calls write (restored before each run, compared after); flags: the int32 error
    words among them.  partial: windows the calls fill only in part (not compared: their unwritten bytes hold what the
    buffer held)."""
    init = [t.clone() for t in state]
    compared = [k for k in sizes if k != "ws" and k not in partial]

    def go(canary):
        for t, s in zip(state, init):
            t.copy_(s)
        lay = _lay(sizes, canary)
        win = {k: v for k, (_, v) in lay.items()}
        ws_bytes = (sizes["ws"] if canary else lay["ws"][0].numel()) if "ws" in sizes else 0
        statuses = [run(win, ws_bytes) for _, run in calls]
        assert all(st == 0 for st in statuses), (statuses, L.recnn_b200_last_error())
        torch.cuda.synchronize()
        return lay, [_bytes(win[k]) for k in compared] + [_bytes(t) for t in state]

    _, want = go(False)
    lay, got = go(True)
    for name, (buf, _) in lay.items():
        assert bool((buf[:OFFSET] == CANARY).all()), "%s: write before the window" % name
        tail = (buf[OFFSET + sizes[name]:] != CANARY).nonzero()
        assert tail.numel() == 0, "%s: write %d bytes past the reported size" % (name, int(tail[0]) + 1)
    names = compared + ["state %d" % i for i in range(len(state))]
    for name, w, g in zip(names, want, got):
        assert torch.equal(w, g), "%s differs from the run on generous zero-filled buffers" % name
    if "ws" in sizes:
        _check_refused(sizes, calls, state, init, flags)


def _check_refused(sizes, calls, state, init, flags):
    """every call that takes the workspace, on one byte less: refused before anything runs"""
    for t, s in zip(state, init):
        t.copy_(s)
    for f in flags:
        f.fill_(SENTINEL)
    lay = _lay({k: n for k, n in sizes.items() if k != "ws"}, True)
    win = {k: v for k, (_, v) in lay.items()}
    short = [run for takes_ws, run in calls if takes_ws]
    check_too_small(sizes["ws"], lambda ptr, nbytes: [run(dict(win, ws=_At(ptr)), nbytes) for run in short])
    torch.cuda.synchronize()
    for f in flags:
        assert f.view(torch.int32).tolist() == [SENTINEL] * f.numel(), "the error flag was written by a refused call"
    for name, (buf, _) in lay.items():
        assert bool((buf == CANARY).all()), "%s was written by a refused call" % name


def _ptr(w, name):
    return w[name].data_ptr()


# ---------------------------------------------------------------- item-set tables and exclusion lists
def set_table(n, items, seed):
    """(set_ids, n_set_ids, set_offsets, n_sets, row_set) on the device: row 0's set is longer than kSetStage (the
    global-memory search; repeated ids when the vocabulary is smaller), rows share sets, every fifth row has none"""
    rng = np.random.default_rng(seed)
    lists = [np.sort(rng.integers(0, items, STAGE + 3))]
    lists += [np.sort(rng.choice(items, m, replace=False)) for m in (1, 7, min(300, items))]
    row_set = np.array([-1 if r % 5 == 4 else r % len(lists) for r in range(n)], dtype=np.int64)
    offsets = np.concatenate([[0], np.cumsum([len(x) for x in lists])]).astype(np.int64)
    ids = np.concatenate(lists).astype(np.int64)
    dev = [torch.from_numpy(x).to(DEV) for x in (ids, offsets, row_set)]
    return dev[0], len(ids), dev[1], len(lists), dev[2]


def set_args(t):
    ids, n_ids, offsets, n_sets, row_set = t
    return ids.data_ptr(), n_ids, offsets.data_ptr(), n_sets, row_set.data_ptr()


def exclude_list(n, items, seed, width=5):
    rng = np.random.default_rng(seed)
    ex = rng.integers(0, items, (n, width))
    ex[rng.random((n, width)) < 0.3] = -1
    return torch.from_numpy(ex.astype(np.int64)).to(DEV), width


def _flag():
    return torch.zeros(1, dtype=torch.int32, device=DEV)


# ---------------------------------------------------------------- retrieval
# (queries, items, dim, metric): above 65,536 items a slab is 128 query rows, so 130 queries take two slabs that reuse
# the scores and the candidate partials; dim 32 runs the tensor-core GEMM, dim 13 the CUDA-core one
RETRIEVAL = [(130, 70001, 32, _lib.METRIC_L2), (130, 70001, 13, _lib.METRIC_COS), (9, 1000, 32, _lib.METRIC_IP)]


def _retrieval_case(nq, items, dim, metric):
    torch.manual_seed(items + dim)
    table, queries = torch.randn(items, dim, device=DEV), torch.randn(nq, dim, device=DEV)
    norms = None
    if metric != _lib.METRIC_IP:
        norms = torch.empty(items, device=DEV)
        _lib.check(L.recnn_item_norms(table.data_ptr(), items, dim, metric, norms.data_ptr(), _lib.stream_ptr()))
    return table, queries, norms


@pytest.mark.parametrize("k", KS)
@pytest.mark.parametrize("nq,items,dim,metric", RETRIEVAL)
def test_retrieval_topk_sets(nq, items, dim, metric, k):
    table, queries, norms = _retrieval_case(nq, items, dim, metric)
    sets, flag = set_table(nq, items, dim), _flag()

    def run(w, nbytes):
        return L.recnn_retrieve_topk_sets(queries.data_ptr(), nq, dim, table.data_ptr(), items, _lib.ptr(norms), metric,
                                          k, *set_args(sets), _ptr(w, "ids"), _ptr(w, "dist"), flag.data_ptr(),
                                          _ptr(w, "ws"), nbytes, _lib.stream_ptr())
    sizes = dict(ws=L.recnn_retrieve_workspace_bytes(nq, items, k), ids=nq * k * 8, dist=nq * k * 4)
    check_windows(sizes, [(True, run)], [flag], [flag])


@pytest.mark.parametrize("nq,items,dim,metric", RETRIEVAL)
def test_retrieval_rank(nq, items, dim, metric):
    table, queries, norms = _retrieval_case(nq, items, dim, metric)
    sets, flag = set_table(nq, items, dim + 1), _flag()
    target = torch.randint(0, items, (nq,), device=DEV)
    head = (queries.data_ptr(), nq, dim, table.data_ptr(), items, _lib.ptr(norms), metric, target.data_ptr())

    def rank(w, nbytes):
        return L.recnn_retrieve_rank(*head, _ptr(w, "rank"), flag.data_ptr(), _ptr(w, "ws"), nbytes, _lib.stream_ptr())

    def rank_sets(w, nbytes):
        return L.recnn_retrieve_rank_sets(*head, *set_args(sets), _ptr(w, "rank"), flag.data_ptr(), _ptr(w, "ws"),
                                          nbytes, _lib.stream_ptr())
    sizes = dict(ws=L.recnn_retrieve_rank_workspace_bytes(nq, items), rank=nq * 8)
    for run in (rank, rank_sets):
        check_windows(sizes, [(True, run)], [flag], [flag])


# ---------------------------------------------------------------- slate distances (outputs only)
@pytest.mark.parametrize("k", KS)
@pytest.mark.parametrize("dim", [13, 132])      # unaligned rows (scalar staging); two 128-dim slices with cp.async
def test_slate_distances(dim, k):
    n, items = 37, 500
    torch.manual_seed(dim * 100 + k)
    table = torch.randn(items, dim, device=DEV)
    ids = torch.randint(0, items, (n, k), device=DEV)
    ids[torch.rand(n, k, device=DEV) < 0.2] = -1
    flag = _flag()
    for metric in (0, 1):
        def run(w, nbytes):
            return L.recnn_slate_distances(ids.data_ptr(), n, k, table.data_ptr(), items, dim, metric, _ptr(w, "mean"),
                                           _ptr(w, "min"), _ptr(w, "count"), _ptr(w, "matrix"), flag.data_ptr(),
                                           _lib.stream_ptr())
        check_windows(dict(mean=n * 4, min=n * 4, count=n * 4, matrix=n * k * k * 4), [(False, run)], [flag])


# ---------------------------------------------------------------- critic serving
# (S, A, H, items, rows, chunk): the tensor cores, every item in three 4,096-wide chunks (the default); H % 4 != 0 runs
# every GEMM on the CUDA cores, in three 1,000-wide chunks.  Candidates: 2,100 per row, more than one 2,048-id tile of
# the repeat check.
CRITIC = [(52, 16, 64, 9000, 10, 0), (37, 13, 30, 2500, 9, 1000)]
N_CAND = 2100


@pytest.mark.parametrize("with_sets", [False, True])
@pytest.mark.parametrize("mode", ["candidates", "all items"])
@pytest.mark.parametrize("S,A,H,items,n,chunk", CRITIC)
def test_critic_serving(S, A, H, items, n, chunk, mode, with_sets):
    torch.manual_seed(S + items)
    critic = recnn_b200.nn.Critic(S, A, H).to(DEV).eval()
    d, params = _lib.Dims(S, A, H, 0), param_arena(critic).data_ptr()
    state, table = torch.randn(n, S, device=DEV), torch.randn(items, A, device=DEV)
    rng = np.random.default_rng(items)
    cand, M = None, 0
    if mode == "candidates":
        c = np.stack([rng.permutation(items)[:N_CAND] for _ in range(n)])
        c[rng.random(c.shape) < 0.1] = -1
        cand, M = torch.from_numpy(c.astype(np.int64)).to(DEV), N_CAND
    sets = set_table(n, items, S) if with_sets else None
    excl = set_args(sets) if sets else (None, 0, None, 0, None)
    target = torch.from_numpy(rng.integers(0, items, n).astype(np.int64)).to(DEV)
    flag = _flag()
    head = (d, params, state.data_ptr(), n, table.data_ptr(), items, _lib.ptr(cand), M)
    for k in KS:
        def topk(w, nbytes):
            return L.recnn_critic_topk(*head, k, *excl, chunk, _ptr(w, "values"), _ptr(w, "ids"), flag.data_ptr(),
                                       _ptr(w, "ws"), nbytes, _lib.stream_ptr())
        sizes = dict(ws=L.recnn_critic_serve_workspace_bytes(d, n, M, items, k, chunk), values=n * k * 4, ids=n * k * 8)
        check_windows(sizes, [(True, topk)], [flag], [flag])

    def rank(w, nbytes):
        return L.recnn_critic_rank(*head, target.data_ptr(), *excl, chunk, _ptr(w, "rank"), flag.data_ptr(),
                                   _ptr(w, "ws"), nbytes, _lib.stream_ptr())
    sizes = dict(ws=L.recnn_critic_serve_workspace_bytes(d, n, M, items, 0, chunk), rank=n * 8)
    check_windows(sizes, [(True, rank)], [flag], [flag])


# ---------------------------------------------------------------- the policy's top-k and sampled slates
@pytest.mark.parametrize("k", KS)
@pytest.mark.parametrize("S,H,I,n,chunk", DISCRETE)
def test_policy_topk_and_slates(S, H, I, n, chunk, k):
    m, state = _discrete(S, H, I, n)[:2]
    d, p, s = m.dims, param_arena(m).data_ptr(), state.data_ptr()
    sets, (ex, E), flag = set_table(n, I, S), exclude_list(n, I, H), _flag()
    seed, row_offset = 99, 12345

    def topk(w, nbytes):
        return L.recnn_discrete_topk(d, p, s, n, k, ex.data_ptr(), E, chunk, _ptr(w, "values"), _ptr(w, "ids"),
                                     flag.data_ptr(), _ptr(w, "ws"), nbytes, _lib.stream_ptr())

    def topk_sets(w, nbytes):
        return L.recnn_discrete_topk_sets(d, p, s, n, k, *set_args(sets), chunk, _ptr(w, "values"), _ptr(w, "ids"),
                                          flag.data_ptr(), _ptr(w, "ws"), nbytes, _lib.stream_ptr())

    def sample(w, nbytes):
        return L.recnn_discrete_sample_topk(d, p, s, n, k, ex.data_ptr(), E, seed, row_offset, chunk, _ptr(w, "values"),
                                            _ptr(w, "ids"), flag.data_ptr(), _ptr(w, "ws"), nbytes, _lib.stream_ptr())

    def sample_sets(w, nbytes):
        return L.recnn_discrete_sample_topk_sets(d, p, s, n, k, *set_args(sets), seed, row_offset, chunk,
                                                 _ptr(w, "values"), _ptr(w, "ids"), flag.data_ptr(), _ptr(w, "ws"),
                                                 nbytes, _lib.stream_ptr())
    sizes = dict(ws=L.recnn_discrete_topk_workspace_bytes(d, n, k, chunk), values=n * k * 4, ids=n * k * 8)
    for run in (topk, topk_sets, sample, sample_sets):
        check_windows(sizes, [(True, run)], [flag], [flag])


@pytest.mark.parametrize("k", KS)
@pytest.mark.parametrize("S,H,I,n,chunk", DISCRETE)
def test_sharded_topk_and_slates(S, H, I, n, chunk, k):
    """world 1: the rank's record window, copied into the gathered window the finish reads"""
    m, state = _discrete(S, H, I, n)[:2]
    d, p, s, vs = m.dims, param_arena(m).data_ptr(), state.data_ptr(), _lib.VocabShard(0, I, 0, 1)
    sets, (ex, E) = set_table(n, I, S), exclude_list(n, I, H)
    flag, finish_flag = _flag(), _flag()
    seed, row_offset = 7, 3
    ws = L.recnn_discrete_topk_workspace_bytes(d, n, k, chunk)
    outs = dict(values=n * k * 4, ids=n * k * 8)

    def shard(w, nbytes):
        return L.recnn_discrete_shard_topk(d, vs, p, s, n, k, ex.data_ptr(), E, chunk, _ptr(w, "record"),
                                           _ptr(w, "ws"), nbytes, _lib.stream_ptr())

    def shard_sets(w, nbytes):
        return L.recnn_discrete_shard_topk_sets(d, vs, p, s, n, k, *set_args(sets), chunk, _ptr(w, "record"),
                                                flag.data_ptr(), _ptr(w, "ws"), nbytes, _lib.stream_ptr())

    def finish(excl):
        def run(w, nbytes):
            return L.recnn_discrete_shard_topk_finish(d, vs, _ptr(w, "gathered"), n, k, *excl, _ptr(w, "values"),
                                                      _ptr(w, "ids"), finish_flag.data_ptr(), _lib.stream_ptr())
        return False, run

    def sample(w, nbytes):
        return L.recnn_discrete_shard_sample_topk(d, vs, p, s, n, k, ex.data_ptr(), E, seed, row_offset, chunk,
                                                  _ptr(w, "record"), _ptr(w, "ws"), nbytes, _lib.stream_ptr())

    def sample_sets(w, nbytes):
        return L.recnn_discrete_shard_sample_topk_sets(d, vs, p, s, n, k, *set_args(sets), seed, row_offset, chunk,
                                                       _ptr(w, "record"), flag.data_ptr(), _ptr(w, "ws"), nbytes,
                                                       _lib.stream_ptr())

    def sample_finish(excl):
        def run(w, nbytes):
            return L.recnn_discrete_shard_sample_topk_finish(d, vs, _ptr(w, "gathered"), n, k, *excl, seed,
                                                             _ptr(w, "values"), _ptr(w, "ids"), finish_flag.data_ptr(),
                                                             _lib.stream_ptr())
        return False, run
    dense, none = (ex.data_ptr(), E), (None, 0)
    rec = L.recnn_vocab_topk_record_floats(n, k) * 4
    for first, last in ((shard, finish(dense)), (shard_sets, finish(none))):
        check_windows(dict(ws=ws, record=rec, gathered=rec, **outs), [(True, first), _gather("record", "gathered"), last],
                      [flag, finish_flag], [flag, finish_flag])
    rec = L.recnn_vocab_sample_topk_record_floats(n, k) * 4
    for first, last in ((sample, sample_finish(dense)), (sample_sets, sample_finish(none))):
        check_windows(dict(ws=ws, record=rec, gathered=rec, **outs), [(True, first), _gather("record", "gathered"), last],
                      [flag, finish_flag], [flag, finish_flag])


# ---------------------------------------------------------------- ranks and log pi
@pytest.mark.parametrize("S,H,I,n,chunk", DISCRETE)
def test_policy_rank_and_log_prob(S, H, I, n, chunk):
    m, state, action = _discrete(S, H, I, n)[:3]
    d, p, s, t = m.dims, param_arena(m).data_ptr(), state.data_ptr(), action.data_ptr()
    sets, flag = set_table(n, I, S), _flag()
    ws = L.recnn_discrete_rank_workspace_bytes(d, n, chunk)

    def rank(w, nbytes):
        return L.recnn_discrete_rank(d, p, s, t, n, chunk, _ptr(w, "rank"), _ptr(w, "log_prob"), flag.data_ptr(),
                                     _ptr(w, "ws"), nbytes, _lib.stream_ptr())

    def rank_sets(w, nbytes):
        return L.recnn_discrete_rank_sets(d, p, s, t, n, *set_args(sets), chunk, _ptr(w, "rank"), _ptr(w, "log_prob"),
                                          flag.data_ptr(), _ptr(w, "ws"), nbytes, _lib.stream_ptr())

    def log_prob(w, nbytes):
        return L.recnn_discrete_log_prob(d, p, s, t, n, chunk, _ptr(w, "log_prob"), flag.data_ptr(), _ptr(w, "ws"),
                                         nbytes, _lib.stream_ptr())
    for run in (rank, rank_sets):
        check_windows(dict(ws=ws, rank=n * 8, log_prob=n * 4), [(True, run)], [flag], [flag])
    check_windows(dict(ws=ws, log_prob=n * 4), [(True, log_prob)], [flag], [flag])


@pytest.mark.parametrize("S,H,I,n,chunk", DISCRETE)
def test_sharded_rank_and_log_prob(S, H, I, n, chunk):
    """world 1: stats record -> gathered -> count record -> gathered -> finish; and the stats records of both pass-1
    phases -> vocab_log_prob_finish"""
    m, state, action = _discrete(S, H, I, n)[:3]
    d, p, s, t = m.dims, param_arena(m).data_ptr(), state.data_ptr(), action.data_ptr()
    vs = _lib.VocabShard(0, I, 0, 1)
    sets, flag, finish_flag = set_table(n, I, S), _flag(), _flag()
    ws = L.recnn_discrete_rank_workspace_bytes(d, n, chunk)
    stats, counts = L.recnn_vocab_record_floats(n) * 4, L.recnn_vocab_rank_record_floats(n) * 4

    def rank_stats(w, nbytes):
        return L.recnn_discrete_shard_rank_stats(d, vs, p, s, t, n, chunk, _ptr(w, "stats"), _ptr(w, "ws"), nbytes,
                                                 _lib.stream_ptr())

    def count(w, nbytes):
        return L.recnn_discrete_shard_rank(d, vs, p, t, n, chunk, _ptr(w, "g_stats"), _ptr(w, "counts"),
                                           _ptr(w, "ws"), nbytes, _lib.stream_ptr())

    def count_sets(w, nbytes):
        return L.recnn_discrete_shard_rank_sets(d, vs, p, t, n, *set_args(sets), chunk, _ptr(w, "g_stats"),
                                                _ptr(w, "counts"), flag.data_ptr(), _ptr(w, "ws"), nbytes,
                                                _lib.stream_ptr())

    def finish(w, nbytes):
        return L.recnn_discrete_shard_rank_finish(d, vs, _ptr(w, "g_stats"), _ptr(w, "g_counts"), t, n,
                                                  _ptr(w, "rank"), _ptr(w, "log_prob"), finish_flag.data_ptr(),
                                                  _lib.stream_ptr())

    def log_prob_finish(w, nbytes):
        return L.recnn_vocab_log_prob_finish(vs, _ptr(w, "g_stats"), t, n, _ptr(w, "log_prob"), finish_flag.data_ptr(),
                                             _lib.stream_ptr())
    sizes = dict(ws=ws, stats=stats, g_stats=stats, counts=counts, g_counts=counts, rank=n * 8, log_prob=n * 4)
    for second in (count, count_sets):
        check_windows(sizes, [(True, rank_stats), _gather("stats", "g_stats"), (True, second),
                              _gather("counts", "g_counts"), (False, finish)], [flag, finish_flag], [flag, finish_flag])
    check_windows(dict(ws=ws, stats=stats, g_stats=stats, log_prob=n * 4),
                  [(True, rank_stats), _gather("stats", "g_stats"), (False, log_prob_finish)], [finish_flag],
                  [finish_flag])

    # the policy gradient's stats phase writes the same record from a float scratch (no byte count to refuse)
    def grad_stats(w, nbytes):
        return L.recnn_reinforce_shard_stats(d, vs, p, s, t, n, chunk, _ptr(w, "stats"), _ptr(w, "scratch"),
                                             _lib.stream_ptr())
    check_windows(dict(scratch=L.recnn_reinforce_scratch_floats(d, n, chunk) * 4, stats=stats, g_stats=stats,
                       log_prob=n * 4),
                  [(False, grad_stats), _gather("stats", "g_stats"), (False, log_prob_finish)], [finish_flag],
                  [finish_flag], partial=["scratch"])


# ---------------------------------------------------------------- the behaviour policy beta
def _beta(S, I, n):
    torch.manual_seed(S + I)
    beta = recnn_b200.nn.Beta(S, I).to(DEV)
    state = torch.randn(n, S, device=DEV)
    action = torch.randint(0, I, (n,), device=DEV)
    return beta, state, action


@pytest.mark.parametrize("S,H,I,n,chunk", DISCRETE)
def test_beta_log_prob(S, H, I, n, chunk):
    beta, state, action = _beta(S, I, n)
    d, p, vs = beta.dims, param_arena(beta).data_ptr(), _lib.VocabShard(0, I, 0, 1)
    flag = _flag()
    ws = L.recnn_beta_log_prob_workspace_bytes(d, n, chunk)
    head = (d, p, state.data_ptr(), S, action.data_ptr(), n, chunk)

    def log_prob(w, nbytes):
        return L.recnn_beta_log_prob(*head, _ptr(w, "log_prob"), flag.data_ptr(), _ptr(w, "ws"), nbytes,
                                     _lib.stream_ptr())

    def stats(w, nbytes):
        return L.recnn_beta_shard_log_prob_stats(d, vs, *head[1:], _ptr(w, "stats"), _ptr(w, "ws"), nbytes,
                                                 _lib.stream_ptr())

    def finish(w, nbytes):
        return L.recnn_vocab_log_prob_finish(vs, _ptr(w, "g_stats"), action.data_ptr(), n, _ptr(w, "log_prob"),
                                             flag.data_ptr(), _lib.stream_ptr())
    check_windows(dict(ws=ws, log_prob=n * 4), [(True, log_prob)], [flag], [flag])
    rec = L.recnn_vocab_record_floats(n) * 4
    check_windows(dict(ws=ws, stats=rec, g_stats=rec, log_prob=n * 4),
                  [(True, stats), _gather("stats", "g_stats"), (False, finish)], [flag], [flag])


@pytest.mark.parametrize("S,H,I,n,chunk", DISCRETE)
def test_beta_shard_phases(S, H, I, n, chunk):
    """world 1: begin -> record -> gathered -> rows -> record -> gathered -> end, probs_out in a window of its own"""
    beta, state, action = _beta(S, I, n)
    o, vs = beta.optim, _lib.VocabShard(0, I, 0, 1)
    loss, error = torch.zeros((), device=DEV), _flag()
    a = _lib.BetaArgs()
    a.dims, a.n_rows, a.chunk_items = beta.dims, n, chunk
    a.net, a.optim = o.c_net(beta), o.c_optim()
    a.state, a.state_ld, a.action = state.data_ptr(), S, action.data_ptr()
    a.loss, a.error = loss.data_ptr(), error.data_ptr()
    state_t = [loss, error, param_arena(beta), grad_arena(beta)]
    state_t += [t for t in (o._m, o._v, o._t, o._slow) if t is not None]

    def bind(w, nbytes):
        a.workspace, a.workspace_bytes, a.probs_out = _ptr(w, "ws"), nbytes, _ptr(w, "probs")

    def begin(w, nbytes):
        bind(w, nbytes)
        return L.recnn_beta_shard_begin(a, vs, _ptr(w, "rec1"), _lib.stream_ptr())

    def rows(w, nbytes):
        bind(w, nbytes)
        return L.recnn_beta_shard_rows(a, vs, _ptr(w, "g1"), _ptr(w, "rec2"), _lib.stream_ptr())

    def end(w, nbytes):
        bind(w, nbytes)
        return L.recnn_beta_shard_end(a, vs, _ptr(w, "g2"), _lib.stream_ptr())
    rec = L.recnn_vocab_record_floats(n) * 4
    sizes = dict(ws=L.recnn_beta_workspace_bytes(beta.dims, n, chunk), probs=n * I * 4, rec1=rec, g1=rec, rec2=rec,
                 g2=rec)
    check_windows(sizes, [(True, begin), _gather("rec1", "g1"), (True, rows), _gather("rec2", "g2"), (True, end)],
                  state_t, [error])


# ---------------------------------------------------------------- the item-id critic, data parallel at world 1
@pytest.mark.parametrize("S,H,I,n,chunk", DISCRETE)
def test_item_id_critic_data_parallel(S, H, I, n, chunk):
    """dp_begin -> grad message (the all-reduce is the identity) and record -> gathered -> dp_end, with a record
    capacity above the rank's rows; the record's rows past n_rows are never written, so it is not compared"""
    rk, _, state = _critic_rank(S, H, I, n, chunk, train=chunk == 128)
    a, record_rows = rk.args, n + 3
    errors = rk.losses.view(torch.int32)[4:5]

    def begin(w, nbytes):
        a.workspace, a.workspace_bytes = _ptr(w, "ws"), nbytes
        return L.recnn_discrete_value_dp_begin(a, 0, n, record_rows, _ptr(w, "grad"), _ptr(w, "record"),
                                               _lib.stream_ptr())

    def end(w, nbytes):
        a.workspace, a.workspace_bytes = _ptr(w, "ws"), nbytes
        return L.recnn_discrete_value_dp_end(a, 0, n, 1, record_rows, _ptr(w, "grad"), _ptr(w, "gathered"),
                                             _lib.stream_ptr())
    rec = L.recnn_discrete_value_dp_record_floats(a.dims, record_rows) * 4
    sizes = dict(ws=L.recnn_discrete_value_dp_workspace_bytes(a.dims, a.policy_dims, n, n, a.chunk_items),
                 grad=L.recnn_discrete_value_dp_grad_floats(a.dims) * 4, record=rec, gathered=rec)
    check_windows(sizes, [(True, begin), _gather("record", "gathered"), (True, end)], state, [errors],
                  partial=["record", "gathered"])
