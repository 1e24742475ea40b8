"""Host-side checks of off-policy estimation: the log-prob entry points in the header, the library and the ctypes
table, their workspace sizes; the refusals of DiscreteActor.log_prob, Beta.log_prob and off_policy_estimates before
any device work; the estimators against numpy, their edge cases and a simulated bandit; and their all-reduce through a
gloo world of 2.  No kernel is launched."""
from __future__ import annotations

import math
import os
import re
import socket

import numpy as np
import pytest
import torch

import recnn_b200
from recnn_b200 import _lib
from recnn_b200.utils.metrics import off_policy_estimates
from tests import _ope_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW_SYMBOLS = ("recnn_discrete_log_prob", "recnn_vocab_log_prob_finish", "recnn_beta_log_prob_workspace_bytes",
               "recnn_beta_log_prob", "recnn_beta_shard_log_prob_stats")


def test_new_symbols_in_header_library_and_ctypes_table():
    with open(os.path.join(ROOT, "include", "recnn_b200.h")) as fh:
        declared = set(re.findall(r"RECNN_API\s+[\w\s\*]+?\b(recnn_\w+)\s*\(", fh.read()))
    L = _lib.lib()
    for name in NEW_SYMBOLS:
        assert name in declared and name in _lib.SIGNATURES, name
        assert getattr(L, name) is not None
    assert declared <= set(_lib.SIGNATURES), sorted(declared - set(_lib.SIGNATURES))
    assert L.recnn_b200_abi_version() == 3


def test_beta_log_prob_workspace_is_one_chunk_and_no_gradient_scratch():
    L = _lib.lib()
    d = _lib.BetaDims(2570, 1 << 20, (0, 0))
    for n, chunk in [(2048, 131072), (128, 1 << 20), (16384, 16384)]:
        ws = L.recnn_beta_log_prob_workspace_bytes(d, n, chunk)
        assert n * chunk * 4 < ws <= n * (2572 + chunk + 3) * 4 + 8 * 256
        assert ws < L.recnn_beta_workspace_bytes(d, n, chunk)
    assert L.recnn_beta_log_prob_workspace_bytes(d, 16, 100) == 0                  # chunk refused
    assert L.recnn_beta_log_prob_workspace_bytes(d, 0, 128) == 0


def test_c_refusals_before_device_work():
    L = _lib.lib()
    k0 = L.recnn_b200_launch_count()
    d = _lib.DiscreteDims(6, 8, 300, 0)
    bd = _lib.BetaDims(6, 300, (0, 0))
    fake = 256                                  # never dereferenced: every call below is refused by its checks
    assert L.recnn_discrete_log_prob(d, fake, fake, fake, 4, 100, fake, fake, fake, 1 << 20, None) != 0
    assert L.recnn_discrete_log_prob(d, fake, fake, fake, 4, 300, fake, fake, fake, 16, None) != 0       # workspace
    assert L.recnn_discrete_log_prob(d, fake, None, fake, 4, 300, fake, fake, fake, 1 << 20, None) != 0
    assert L.recnn_beta_log_prob(bd, fake, fake, 6, fake, 4, 100, fake, fake, fake, 1 << 20, None) != 0
    assert L.recnn_beta_log_prob(bd, fake, fake, 5, fake, 4, 300, fake, fake, fake, 1 << 20, None) != 0  # state_ld
    assert L.recnn_beta_log_prob(bd, fake, fake, 6, fake, 4, 300, fake, fake, fake, 16, None) != 0
    bad = _lib.VocabShard(0, 300, 2, 2)                                        # rank outside the world
    assert L.recnn_beta_shard_log_prob_stats(bd, bad, fake, fake, 6, fake, 4, 300, fake, fake, 1 << 20, None) != 0
    assert L.recnn_vocab_log_prob_finish(bad, fake, fake, 4, fake, fake, None) != 0
    assert L.recnn_vocab_log_prob_finish(_lib.VocabShard(300, 300, 0, 1), fake, fake, 4, fake, fake, None) != 0
    assert L.recnn_vocab_log_prob_finish(_lib.VocabShard(0, 300, 0, 1), fake, fake, 0, fake, fake, None) != 0
    assert L.recnn_b200_launch_count() == k0


def test_module_refusals_happen_before_device_work():
    L = _lib.lib()
    torch.manual_seed(0)
    m = recnn_b200.nn.DiscreteActor(6, 10, 8)
    b = recnn_b200.nn.Beta(6, 10)
    st = torch.zeros(3, 6)
    a = torch.tensor([1, 2, 3])
    k0 = L.recnn_b200_launch_count()
    for net in (m, b):
        with pytest.raises(ValueError, match="state"):
            net.log_prob(torch.zeros(3, 5), a)
        with pytest.raises(ValueError):
            net.log_prob(st, torch.tensor([1, 2]))
        with pytest.raises(_lib.RecnnError, match="CUDA only"):
            net.log_prob(st, a)
    for bad in (torch.tensor([[1, 2, 3]]), torch.tensor([1.0, 2.0, 3.0]), torch.tensor([True, False, True]),
                [1, 2, 3]):
        with pytest.raises(ValueError, match="action"):
            m.log_prob(st, bad)
    with pytest.raises(ValueError, match="one-hot"):
        b.log_prob(st, torch.zeros(3, 9))
    with pytest.raises(_lib.RecnnError, match="CUDA only"):
        b.log_prob(st, torch.eye(10)[:3])                                     # the one-hot form is accepted
    assert L.recnn_b200_launch_count() == k0


# ----------------------------------------------------------------------------- the estimators
def _case(n, seed):
    rng = np.random.default_rng(seed)
    lp_b = np.log(rng.uniform(1e-4, 0.2, n))
    lp_p = np.log(rng.uniform(1e-5, 0.5, n))
    r = rng.integers(0, 6, n).astype(np.float64)
    return lp_p, lp_b, r


@pytest.mark.parametrize("K", [1, 2, 10])
def test_estimators_against_numpy(K):
    lp_p, lp_b, r = _case(500, K)
    for clip in (None, 3.0):
        got = off_policy_estimates(torch.from_numpy(lp_p).float(), torch.from_numpy(lp_b).float(),
                                   torch.from_numpy(r).float(), K=K, clip=clip)
        want = O.estimates(np.float32(lp_p), np.float32(lp_b), np.float32(r), K=K, clip=clip)
        assert set(got) == set(want)
        for k in want:
            assert got[k] == pytest.approx(want[k], rel=1e-10), (k, got[k], want[k])
    assert got["n"] == 500 and 0 < got["clipped_share"] < 1


def test_equal_log_probs_give_unit_weights():
    lp_p, _, r = _case(333, 4)
    got = off_policy_estimates(torch.from_numpy(lp_p), torch.from_numpy(lp_p), torch.from_numpy(r))
    assert got["ips"] == got["snips"] == pytest.approx(r.mean(), rel=1e-15)
    assert got["logged_reward"] == pytest.approx(r.mean(), rel=1e-15)
    assert got["ess"] == pytest.approx(333, rel=1e-15) and got["max_weight"] == 1.0
    assert got["ips_stderr"] == pytest.approx(r.std(ddof=1) / math.sqrt(333), rel=1e-12)


def test_top_k_weight_is_stable_for_improbable_items():
    """log pi = -20 with K = 10: alpha_K = 1 - (1 - pi)^10 = 10 pi (1 - 4.5 pi + ...), which 1 - (1 - pi)**K would
    lose entirely in float64 rounding of 1 - pi."""
    lp = torch.full((4,), -20.0, dtype=torch.float64)
    got = off_policy_estimates(lp, torch.zeros(4, dtype=torch.float64), torch.ones(4, dtype=torch.float64), K=10)
    pi = math.exp(-20.0)
    want = 10 * pi * (1 - 4.5 * pi)
    assert got["ips"] == pytest.approx(want, rel=1e-12)
    tiny = off_policy_estimates(torch.tensor([-800.0]), torch.tensor([-799.0]), torch.tensor([1.0]), K=3)
    assert tiny["ips"] == pytest.approx(3 * math.exp(-1.0), rel=1e-12)          # pi underflows float64
    one = off_policy_estimates(torch.tensor([0.0, 1e-7]), torch.tensor([0.0, 0.0]), torch.tensor([1.0, 1.0]), K=4)
    assert one["ips"] == 1.0                                                     # pi = 1 is in every slate


def test_simulated_bandit_lands_within_four_standard_errors():
    rng = np.random.default_rng(11)
    items, n = 50, 20000
    beta = rng.dirichlet(np.ones(items))
    beta = 0.5 * beta + 0.5 / items                                   # full support
    pi = rng.dirichlet(np.full(items, 0.3))
    mean_r = rng.uniform(0, 5, items)
    a = rng.choice(items, n, p=beta)
    r = mean_r[a] + rng.normal(0, 1, n)
    for K in (1, 3):
        alpha = 1 - (1 - pi) ** K
        true = (alpha * mean_r).sum()
        got = off_policy_estimates(torch.from_numpy(np.log(pi[a])), torch.from_numpy(np.log(beta[a])),
                                   torch.from_numpy(r), K=K)
        assert abs(got["ips"] - true) < 4 * got["ips_stderr"], (K, got, true)
        assert got["logged_reward"] == pytest.approx((beta * mean_r).sum(), abs=4 * r.std() / math.sqrt(n))
        assert 0 < got["ess"] < n


def test_estimator_refusals():
    x = torch.zeros(4)
    for bad in (torch.zeros(3), torch.zeros(4, 1)):
        with pytest.raises(ValueError):
            off_policy_estimates(x, bad, x)
        with pytest.raises(ValueError):
            off_policy_estimates(x, x, bad)
    for K in (0, -1, 1.5, True, "2"):
        with pytest.raises(ValueError, match="K"):
            off_policy_estimates(x, x, x, K=K)
    for clip in (0, -1.0, float("nan"), True):
        with pytest.raises(ValueError, match="clip"):
            off_policy_estimates(x, x, x, clip=clip)
    for v in (float("nan"), float("inf"), -float("inf")):
        with pytest.raises(ValueError, match="non-finite"):
            off_policy_estimates(torch.tensor([0.0, v]), torch.zeros(2), torch.ones(2))
        with pytest.raises(ValueError, match="non-finite"):
            off_policy_estimates(torch.zeros(2), torch.tensor([v, 0.0]), torch.ones(2))
    empty = off_policy_estimates(torch.zeros(0), torch.zeros(0), torch.zeros(0), clip=2.0)
    assert empty["n"] == 0 and math.isnan(empty["ips"]) and math.isnan(empty["clipped_ips"])


def _gloo_worker(rank, world, port, q):
    import torch.distributed as dist
    dist.init_process_group("gloo", init_method="tcp://127.0.0.1:%d" % port, rank=rank, world_size=world)
    try:
        lp_p, lp_b, r = _case(301, 7)
        part = slice(0, 120) if rank == 0 else slice(120, 301)
        t = lambda x: torch.from_numpy(x[part])
        q.put((rank, off_policy_estimates(t(lp_p), t(lp_b), t(r), K=2, clip=4.0, group=dist.group.WORLD)))
    finally:
        dist.destroy_process_group()


def test_group_all_reduce_over_gloo_equals_one_process():
    import torch.multiprocessing as mp
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_gloo_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    got = dict(q.get(timeout=120) for _ in range(2))
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    lp_p, lp_b, r = _case(301, 7)
    want = off_policy_estimates(torch.from_numpy(lp_p), torch.from_numpy(lp_b), torch.from_numpy(r), K=2, clip=4.0)
    assert want["n"] == 301
    for k in want:
        assert got[0][k] == pytest.approx(want[k], rel=1e-12) and got[1][k] == got[0][k], k
