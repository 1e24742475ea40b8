"""Virtual ranks: W copies of the vocabulary-parallel public API in one process, on one device.

``run_ranks(world, fn)`` calls ``fn(rank)`` on W threads, one at a time: rank 0 runs until its first exchange, then
rank 1, ..., and the last rank to arrive completes the exchange and hands back to rank 0.  Every CUDA call is thus
enqueued in one fixed order on the default stream, and the C library is never entered from two threads at once.  Each
rank gets an ``_Exchange``, the ``comm`` a ``VocabParallel`` uses: ``all_gather`` concatenates the ranks' tensors in rank
order (what recnn_comm_allgather delivers) and ``all_reduce`` sums them in rank order in fp32 (the order
allreduce_kernel sums in).  ``shard`` builds one rank's nets through ``recnn_b200.dist.shard_in_place``.

Also here: the fixtures and helpers the vocabulary-parallel test modules share (a one-rank process group, bit views,
the spawn of W worker processes)."""
from __future__ import annotations

import contextlib
import socket
import threading
import time

import pytest
import torch

from recnn_b200 import dist as D
from recnn_b200.nn.update import reinforce as RF

_local = threading.local()


class RanksError(RuntimeError):
    """The virtual ranks did not make the same exchanges: one returned or raised while others waited in one, their
    tensors differ in size or dtype, or a rank waited longer than the timeout."""


class _Exchange:
    """One virtual rank's communicator: what VocabParallel calls on its ``comm``."""
    capacity = 1 << 62                         # VocabParallel._fit never grows it (growing needs a process group)

    def __init__(self, run, rank):
        self.run, self.rank, self.world = run, rank, run.world

    def all_gather(self, t):
        """[world * numel]: every rank's ``t`` in rank order (or the run's order for this gather), a new tensor."""
        return self.run.exchange(self.rank, "all_gather", t)

    def all_reduce(self, t):
        """In place: rank 0's ``t`` plus each later rank's, in rank order; the same bits on every rank."""
        return self.run.exchange(self.rank, "all_reduce", t)

    def close(self):
        pass


class _Run:
    def __init__(self, world, order, log, timeout):
        self.world, self.order, self.log, self.timeout = world, order or {}, log, timeout
        self.cv = threading.Condition()
        self.turn = 0
        self.posted = []                        # (rank, kind, tensor) of the exchange under way
        self.delivered = [None] * world
        self.finished = set()
        self.broken = None
        self.gathers = 0
        self.cuda = torch.cuda.is_available()
        self.rng = [self._rng_state()] * world
        self.results = [None] * world

    def _rng_state(self):
        return torch.get_rng_state(), (torch.cuda.get_rng_state() if self.cuda else None)

    def _wait(self, r):
        """Until it is rank r's turn (holding the lock); then rank r's RNG state is the process's."""
        deadline = time.monotonic() + self.timeout
        while self.turn != r:
            left = deadline - time.monotonic()
            if left <= 0:
                self.broken = self.broken or "rank %d waited more than %g s for its turn" % (r, self.timeout)
                raise RanksError(self.broken)
            self.cv.wait(left)
        cpu, cuda = self.rng[r]
        torch.set_rng_state(cpu)
        if cuda is not None:
            torch.cuda.set_rng_state(cuda)

    def _hand_off(self, r, to):
        self.rng[r] = self._rng_state()
        self.turn = to
        self.cv.notify_all()

    def _check(self):
        if self.broken is not None:
            raise RanksError(self.broken)

    def exchange(self, r, kind, t):
        with self.cv:
            self._check()
            if self.finished:
                self.broken = "rank(s) %s ended before an %s that rank %d made" % (sorted(self.finished), kind, r)
                raise RanksError(self.broken)
            self.posted.append((r, kind, t))
            if len(self.posted) < self.world:
                self._hand_off(r, r + 1)
            else:
                self._complete()
                self._hand_off(r, 0)
            self._wait(r)
            self._check()
            return self.delivered[r]

    def _complete(self):
        posted, self.posted = self.posted, []
        if len({(k, t.numel(), t.dtype) for _, k, t in posted}) != 1:
            self.broken = "the ranks' exchanges differ: %s" % [(q, k, t.numel(), str(t.dtype)) for q, k, t in posted]
            return
        kind, ts = posted[0][1], [t for _, _, t in posted]
        if kind == "all_gather":
            order = self.order.get(self.gathers, range(self.world))
            self.gathers += 1
            out = torch.cat([ts[q].reshape(-1) for q in order])
            self.delivered = [out.clone() for _ in ts]
        else:
            out = ts[0].clone()
            for t in ts[1:]:
                out += t
            for t in ts:
                t.copy_(out)
            self.delivered = ts
        if self.log is not None:
            self.log.append((kind, out))

    def main(self, r, fn):
        _local.exchange = _Exchange(self, r)
        try:
            with self.cv:
                self._wait(r)
            out = fn(r)
        except BaseException as exc:           # noqa: BLE001 -- handed back to the caller as this rank's outcome
            out = exc
        with self.cv:
            self.results[r] = out
            self.finished.add(r)
            if self.posted and self.broken is None:
                self.broken = "rank %d %s while rank(s) %s wait in an %s" % (
                    r, "raised %r" % out if isinstance(out, BaseException) else "returned",
                    [q for q, _, _ in self.posted], self.posted[0][1])
            rest = [q % self.world for q in range(r + 1, r + self.world) if q % self.world not in self.finished]
            self._hand_off(r, rest[0] if rest else None)


def run_ranks(world, fn, order=None, log=None, timeout=300.0):
    """``[fn(0), ..., fn(world - 1)]``, each entry the rank's result or the exception it raised.  Every rank starts
    from the caller's torch CPU and CUDA generator states and keeps its own (the draws of a same-seeded process); the
    caller's states are restored afterwards.  ``order``: {i: rank order} of the i-th all-gather (0-based), to deliver
    records out of rank order.  ``log``: a list that receives (kind, delivered tensor) per exchange.  When the ranks'
    exchanges do not match, every rank's outcome is a RanksError (or the exception it raised itself)."""
    run = _Run(world, order, log, timeout)
    caller = run._rng_state()
    threads = [threading.Thread(target=run.main, args=(r, fn), daemon=True) for r in range(world)]
    try:
        for t in threads:
            t.start()
        for t in threads:
            t.join(timeout)
            if t.is_alive():
                raise RanksError("a virtual rank did not finish within %g s" % timeout)
    finally:
        torch.set_rng_state(caller[0])
        if caller[1] is not None:
            torch.cuda.set_rng_state(caller[1])
    if run.broken is not None:
        return [out if isinstance(out, BaseException) else RanksError(run.broken) for out in run.results]
    return run.results


def returned(results):
    """The ranks' results; raises the first rank's exception if any rank raised."""
    for out in results:
        if isinstance(out, BaseException):
            raise out
    return results


def exchange():
    """The communicator of the virtual rank running on this thread."""
    return _local.exchange


def _copy(net):
    """A fresh full-size net of ``net``'s class and shape holding its weights (a Beta with its optimizer's lr and
    weight decay), on its device and in its train / eval mode."""
    from recnn_b200.nn.arena import _is_beta, _is_discrete
    from recnn_b200.nn import Beta, Critic, DiscreteActor
    if _is_beta(net):
        g = net.optim.param_groups[0]
        twin = Beta(net.net[0].in_features, net.net[0].out_features, lr=g["lr"], weight_decay=g["weight_decay"])
    elif _is_discrete(net):
        twin = DiscreteActor(net.linear1.in_features, net.linear2.out_features, net.linear1.out_features)
    else:
        twin = Critic(net.linear1.in_features - net._action_dim, net._action_dim, net.linear1.out_features)
    twin.load_state_dict(net.state_dict())
    return twin.to(net.linear1.weight.device if hasattr(net, "linear1") else net.net[0].weight.device).train(
        net.training)


def shard(nets, beta=None):
    """This virtual rank's copies of the full, unsharded ``nets`` ({name: net}, names as in an agent) and ``beta``,
    sharded to the rank's block with shard_in_place on a VocabParallel over its exchange: (nets, beta)."""
    ex = exchange()
    items = nets["policy_net"].linear2.out_features if "policy_net" in nets else beta.net[0].out_features
    lo, hi = D.vocab_shard(items, ex.rank, ex.world)
    local = {k: _copy(net) for k, net in nets.items()}
    local_beta = None if beta is None else _copy(beta)
    D.shard_in_place(local, D.VocabParallel(lo, hi, items, None, ex.rank, ex.world, ex), local_beta)
    return local, local_beta


@contextlib.contextmanager
def chunked(rows, chunk):
    """Calls over ``rows`` rows visit the items in chunks of ``chunk`` (a multiple of 128; None: as configured) while
    the block runs: the logits budget of recnn_b200.nn.update.reinforce._chunk_items, which every chunked call reads."""
    old = RF._LOGITS_BUDGET_BYTES
    if chunk is not None:
        RF._LOGITS_BUDGET_BYTES = rows * 4 * chunk
    try:
        yield
    finally:
        RF._LOGITS_BUDGET_BYTES = old


# ----------------------------------------------------------------------------- shared by the test modules
@pytest.fixture
def one_rank_group(tmp_path):
    """A world-1 NCCL process group on cuda:0."""
    import torch.distributed as dist
    torch.cuda.set_device(0)
    dist.init_process_group("nccl", init_method="file://" + str(tmp_path / "pg"), rank=0, world_size=1,
                            device_id=torch.device("cuda:0"))
    yield
    dist.destroy_process_group()


@pytest.fixture
def one_rank_cpu_group(tmp_path):
    """A world-1 gloo process group."""
    import torch.distributed as dist
    dist.init_process_group("gloo", init_method="file://" + str(tmp_path / "pg"), rank=0, world_size=1)
    yield
    dist.destroy_process_group()


def bits(t):
    """The int32 bit pattern of an fp32 tensor, on the host."""
    return t.detach().contiguous().view(torch.int32).cpu()


def spawn(target, world, *args, items=None, timeout=300):
    """Run ``target(rank, world, port, *args, queue)`` in ``world`` spawned processes (``port``: a free local port for
    the rendezvous) and return the first ``items`` (default: ``world``) objects they put on the queue."""
    import torch.multiprocessing as mp
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=target, args=(r, world, port) + args + (q,)) for r in range(world)]
    for pr in procs:
        pr.start()
    out = [q.get(timeout=timeout) for _ in range(world if items is None else items)]
    for pr in procs:
        pr.join(timeout=timeout)
        assert pr.exitcode == 0
    return out
