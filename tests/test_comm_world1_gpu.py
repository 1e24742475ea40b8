"""The data-parallel all-reduce kernel (csrc/comm.cu) on one GPU, through a world-1 communicator.

For the data-parallel step, allreduce_kernel is a second implementation of the step's serial tail: it sums the
critics' split-K partials (GradSource), applies the built-in optimizer (opt_apply, all kinds) and advances the step
counter, computes the actor's L1 clip coefficient and writes the scaled gradient back, and sums the loss partials
("aux" words); a step without a policy update makes one more launch with n = 0 for the loss alone.  At world 1 every
phase of the kernel runs, with no peer and no cross-process wait, and the single-rank sum is the value itself.  So
wherever the communicator path and the single-GPU path compute the same thing they must agree bit for bit:

  * the collective on its own moves every fp32 bit pattern unchanged (both kernel variants, both epoch parities);
  * TD3's critics never read the online actor (its target policy is never soft-updated, td3.py:136-141): parameters,
    .grad, optimizer state, step counters and value losses are bit-identical at every step;
  * DDPG and TD3 agree bit for bit on step 0 (a policy step) up to the actor's clip coefficient, whose L1 norm is
    summed in a different order; from step 1 DDPG's critic sees that actor through the soft-updated target policy,
    so both runs are held to the float64 oracle instead.

What world 1 does not reach -- slicing across owners, rank-order sums of W > 1 contributions, the double buffering
when one rank is an epoch ahead, the n_rows_global mismatch flag -- is left to the multi-GPU parametrisations of
test_gpu_parity.py::test_data_parallel_equals_reference.  W > 1 is not emulated on one device: the protocol needs
every CTA of every rank resident at once, which one device does not guarantee."""
from __future__ import annotations

import ctypes
import gc
import pickle
import sys

import numpy as np
import pytest
import torch

import recnn_b200
from recnn_b200 import _lib
from recnn_b200.nn.arena import grad_arena, param_arena
from oracle import cases as C
from tests._cuda import build_nets, run_cuda_case
from tests._golden import (assert_oracle_bar, assert_tight_parity, compare_with_golden, load_golden,
                           neutralise_ambiguous_gates, run_oracle_case)
from tests.test_step_shapes_gpu import assert_pads_zero, check_against_oracle, pad_report, prepared, run_sweep

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
POLICY_EVERY = 10                     # C.DDPG_PARAMS["policy_step"] == C.TD3_PARAMS["policy_update"]
SHAPE_ROWS = ("h50", "h100", "h320", "min")
SIMT_ROW = "h320"


# ----------------------------------------------------------------------------- the communicator
class World1Comm:
    """A one-rank peer communicator made through the C ABI (no torch.distributed): create, take the local handle,
    connect with it (a single local handle maps nothing)."""

    def __init__(self, capacity_floats):
        L = _lib.lib()
        self.handle = ctypes.c_void_p()
        _lib.check(L.recnn_comm_create(0, 1, int(capacity_floats), ctypes.byref(self.handle)))
        self.capacity = -(-int(capacity_floats) // 4) * 4       # the library rounds the staging capacity up to 4
        try:
            mine = ctypes.create_string_buffer(L.recnn_comm_handle_bytes())
            _lib.check(L.recnn_comm_local_handle(self.handle, mine))
            _lib.check(L.recnn_comm_connect(self.handle, mine))
        except Exception:
            self.close()
            raise

    @property
    def ptr(self):
        return self.handle.value

    def all_reduce(self, t):
        assert t.is_cuda and t.dtype == torch.float32 and t.is_contiguous()
        _lib.check(_lib.lib().recnn_comm_allreduce(self.handle, t.data_ptr(), t.numel(),
                                                   torch.cuda.current_stream(t.device).cuda_stream))
        return t

    def close(self):
        if self.handle is not None:
            torch.cuda.synchronize()
            _lib.lib().recnn_comm_destroy(self.handle)
            self.handle = None


@pytest.fixture
def open_comm():
    """nets -> a world-1 communicator sized for the largest parameter arena of the nets (the run_cuda_case ``comm``
    hook).  Closed at teardown, once the nets, their engines and graphs are gone and the device is idle."""
    made = []

    def make(nets):
        made.append(World1Comm(max(param_arena(m).numel() for m in nets.values())))
        return made[-1]

    yield make
    gc.collect()
    torch.cuda.synchronize()
    for c in made:
        c.close()


# ----------------------------------------------------------------------------- 1. the collective on its own
def _bits(t):
    return t.detach().contiguous().cpu().view(torch.int32)


def _payload(n, rng):
    """n fp32 words (as int32 on the device) of random bit patterns -- every class: NaNs with payloads, infinities,
    subnormals, both zeros -- led by the special values themselves."""
    special = np.array([0x80000000, 0x00000000, 0x00000001, 0x80000001, 0x007FFFFF, 0x7F800000, 0xFF800000,
                        0x7FC00000, 0x7F800001, 0xFFFFFFFF, 0x7F7FFFFF, 0x00800000], dtype=np.uint32)
    words = rng.integers(0, 1 << 32, n, dtype=np.uint32)
    k = min(n, special.size)
    words[:k] = special[:k]
    return torch.from_numpy(words.view(np.int32)).to(DEV)


CANARY = 0x7FA5A5A5                     # a NaN with a payload


def _canaries(n):
    return torch.full((n,), CANARY, dtype=torch.int32, device=DEV)


def critic_arena_floats(state_dim, action_dim, hidden):
    return param_arena(recnn_b200.nn.Critic(state_dim, action_dim, hidden).to(DEV)).numel()


def test_allreduce_moves_every_bit_pattern_unchanged():
    """recnn_comm_allreduce at world 1 is the identity on the bits: sizes 1..5, 1001, 4096, 4097, a critic arena at
    BASELINE size (S 1290, A 128, H 256) and exactly the staging capacity; VEC = 2 (n even, 8-byte aligned) and
    VEC = 1 (n odd, or a view one float off alignment); NaN canaries around the reduced range stay untouched.  The
    calls run back to back on one stream, so both epoch parities are used many times over."""
    base = critic_arena_floats(1290, 128, 256)
    comm = World1Comm(base + 3)                    # not a multiple of 4: the library rounds up to base + 4
    rng = np.random.default_rng(20261016)
    sizes = (1, 2, 3, 4, 5, 1001, 4096, 4097, base, comm.capacity)
    calls = []
    try:
        for n in sizes:
            for variant in ("own", "offset"):
                x = _payload(n, rng)
                # built and compared as int32 so that no float copy can touch a NaN's bits
                if variant == "own":                 # own allocation (256-byte aligned) with canaries behind it
                    words = torch.cat([x, _canaries(64)])
                    view = words.view(torch.float32)[:n]
                    vec = 2 if n % 2 == 0 else 1
                else:                                # one float in: 4-byte aligned only -> the scalar variant
                    words = torch.cat([_canaries(1), x, _canaries(63)])
                    view = words.view(torch.float32)[1:n + 1]
                    vec = 1
                assert view.is_contiguous()
                before = words.cpu()
                comm.all_reduce(view)
                torch.cuda.synchronize()
                after = words.cpu()
                diff = int((after != before).sum())
                assert diff == 0, "n=%d %s: %d words changed (first at %d)" % (
                    n, variant, diff, int((after != before).nonzero()[0]))
                calls.append((n, vec))
        assert len(calls) >= 6
        assert {v for _, v in calls} == {1, 2}
        assert any(n == comm.capacity and v == 2 for n, v in calls) and any(n == base and v == 2 for n, v in calls)
        # the staging capacity is the limit: one float more is refused before any launch
        over = torch.zeros(comm.capacity + 1, device=DEV)
        L = _lib.lib()
        k0 = L.recnn_b200_launch_count()
        with pytest.raises(_lib.RecnnError, match="capacity"):
            comm.all_reduce(over)
        assert L.recnn_b200_launch_count() == k0
    finally:
        comm.close()


def test_communicator_error_paths():
    """Each refusal raises RecnnError before any device work; destroy(NULL) is a no-op."""
    L = _lib.lib()
    k0 = L.recnn_b200_launch_count()
    for rank, world in ((0, 0), (0, 9), (1, 1), (2, 2), (-1, 1)):
        h = ctypes.c_void_p()
        with pytest.raises(_lib.RecnnError, match="rank/world"):
            _lib.check(L.recnn_comm_create(rank, world, 16, ctypes.byref(h)))
        assert h.value is None, (rank, world)
    assert L.recnn_comm_destroy(None) == 0
    x = torch.zeros(8, device=DEV)
    # all-reduce on a communicator that was never connected
    h = ctypes.c_void_p()
    _lib.check(L.recnn_comm_create(0, 1, 16, ctypes.byref(h)))
    try:
        with pytest.raises(_lib.RecnnError, match="not connected"):
            _lib.check(L.recnn_comm_allreduce(h, x.data_ptr(), 8, torch.cuda.current_stream().cuda_stream))
    finally:
        L.recnn_comm_destroy(h)
    # a second connect
    comm = World1Comm(16)
    try:
        mine = ctypes.create_string_buffer(L.recnn_comm_handle_bytes())
        _lib.check(L.recnn_comm_local_handle(comm.handle, mine))
        with pytest.raises(_lib.RecnnError, match="already connected"):
            _lib.check(L.recnn_comm_connect(comm.handle, mine))
        with pytest.raises(_lib.RecnnError, match="capacity"):
            comm.all_reduce(torch.zeros(17, device=DEV))
        assert L.recnn_b200_launch_count() == k0
        comm.all_reduce(x)                      # still usable after the refusals
        torch.cuda.synchronize()
        assert L.recnn_b200_launch_count() == k0 + 1
        assert torch.equal(x, torch.zeros(8, device=DEV))
    finally:
        comm.close()


# ----------------------------------------------------------------------------- 2. the step, with and without it
def critic_names(algo):
    return ("value_net",) if algo == "ddpg" else ("value_net1", "value_net2")


def engine_of(nets):
    engines = nets["policy_net"].__dict__["_recnn_engines"]
    assert len(engines) == 1
    return next(iter(engines.values()))


class Recorder:
    """run_cuda_case's on_step hook: after every step, the bits of each critic's whole state (parameters, .grad, the
    optimizer's moment / slow-weight arenas and step counter) and value losses; the policy loss; the engine's kernel
    count and whether the step captured a CUDA graph; after step 0, the actor's parameters, .grad and L1 norm."""

    def __init__(self, algo):
        self.algo = algo
        self.critic, self.policy_loss, self.kernels, self.captured = [], [], [], []
        self.actor0 = None
        self._k = self._g = 0

    def __call__(self, step, nets, opts, loss):
        eng = engine_of(nets)
        snap = {}
        for name in critic_names(self.algo):
            o = opts[name.replace("net", "optimizer")]
            snap[name + ".param"] = _bits(param_arena(nets[name]))
            snap[name + ".grad"] = _bits(grad_arena(nets[name]))
            for a in ("_m", "_v", "_slow", "_t"):
                if getattr(o, a) is not None:
                    snap[name + "." + a] = _bits(getattr(o, a))
        for k in loss:
            if k.startswith("value"):
                snap["loss." + k] = np.float32(loss[k])
        self.critic.append(snap)
        self.policy_loss.append(np.float32(loss["policy"]))
        self.kernels.append(eng.kernels - self._k)
        self.captured.append(len(eng.graphs) > self._g)
        self._k, self._g = eng.kernels, len(eng.graphs)
        if step == 0:
            pol = nets["policy_net"]
            self.actor0 = {"param": param_arena(pol).detach().cpu().clone(),
                           "grad": grad_arena(pol).detach().cpu().clone(),
                           "l1": float(eng.losses[3].item()), "t": _bits(opts["policy_optimizer"]._t)}


def _same_bits(a, b):
    if isinstance(a, torch.Tensor):
        return a.shape == b.shape and torch.equal(a, b)
    return np.asarray(a).view(np.int32) == np.asarray(b).view(np.int32)


def _ulps(a, b):
    """Elementwise distance in units in the last place of two fp32 tensors (through the ordered integer line)."""
    def ordered(x):
        i = x.numpy().view(np.int32).astype(np.int64)
        return np.where(i < 0, -(i & 0x7FFFFFFF), i)
    return np.abs(ordered(a) - ordered(b))


def check_comm_against_plain(algo, plain, comm, p_init, max_ulp=1.0):
    """The assertions that tie the communicator run to the single-GPU run on the same inputs.  Returns the actor's
    largest ulp gap after step 0 and the relative gap of the two L1 norms.  ``p_init``: the actor's parameter arena
    before step 0.  ``max_ulp``: the bound on the actor's weights after step 0 (see run_pair)."""
    n = len(plain.critic)
    assert len(comm.critic) == n
    # 1 / 2: TD3's critics at every step, DDPG's at step 0; the policy loss of step 0 (online actor not yet updated)
    for s in range(n if algo == "td3" else 1):
        a, b = plain.critic[s], comm.critic[s]
        assert a.keys() == b.keys()
        for k in a:
            if not _same_bits(a[k], b[k]):
                diff = int((a[k] != b[k]).sum()) if isinstance(a[k], torch.Tensor) else 1
                raise AssertionError("step %d: %s differs with the communicator (%d words)" % (s, k, diff))
    assert _same_bits(plain.policy_loss[0], comm.policy_loss[0]), (plain.policy_loss[0], comm.policy_loss[0])
    # 3: the actor after step 0.  Same raw gradient; the clip coefficient -1 / (||g||_1 + 1e-6) differs only through
    # the order of the L1 sum.  .grad / coef recovers the raw gradient to the two roundings of coef and of the scaling.
    a, b = plain.actor0, comm.actor0
    assert torch.equal(a["t"], b["t"]) and int(a["t"][0]) == 1
    if a["l1"] == 0.0:              # every actor unit gated off (the smallest net): a zero gradient, scaled to zero
        assert b["l1"] == 0.0 and not a["grad"].any() and not b["grad"].any()
        l1_rel = 0.0
    else:
        l1_rel = abs(b["l1"] - a["l1"]) / abs(a["l1"])
        assert l1_rel <= 1e-6, (a["l1"], b["l1"])
        for r in (a, b):
            s1 = float(r["grad"].double().abs().sum())
            assert abs(s1 - 1.0) <= 1e-5, s1
        raw_a = a["grad"].double() / (-1.0 / (a["l1"] + 1e-6))
        raw_b = b["grad"].double() / (-1.0 / (b["l1"] + 1e-6))
        assert torch.all((raw_a - raw_b).abs() <= 3e-7 * raw_a.abs()), \
            float(((raw_a - raw_b).abs() / raw_a.abs()).nan_to_num().max())
        if a["l1"] == b["l1"]:
            assert torch.equal(_bits(a["grad"]), _bits(b["grad"]))
    # the weights after step 0, in ulps of the larger of the weight before the step and the two results: where an
    # update nearly cancels a weight the result is far smaller than either, and its own ulp says nothing
    p0 = p_init.numpy().astype(np.float64)
    pa, pb = a["param"].numpy().astype(np.float64), b["param"].numpy().astype(np.float64)
    unit = np.spacing(np.maximum(np.maximum(np.abs(p0), np.abs(pa)), np.abs(pb)).astype(np.float32)).astype(np.float64)
    ulp = float(np.max(np.abs(pa - pb) / unit))
    assert ulp <= max_ulp, (ulp, int(_ulps(a["param"], b["param"]).max()))
    # 5: the communicator path ran.  Per critic the optimizer kernel becomes one all-reduce kernel; on a policy step
    # the actor's L1-clip and optimizer kernels become one all-reduce kernel (step.cu phase_policy_opt); a step
    # without a policy update adds the n = 0 loss exchange (PH_FINISH).  A capture step counts its kernels once as
    # recorded and once for its first replay: those steps are left out.
    assert plain.captured == comm.captured
    seen = set()
    for s in range(n):
        if plain.captured[s]:
            continue
        pol = s % POLICY_EVERY == 0
        assert comm.kernels[s] - plain.kernels[s] == (-1 if pol else 1), (s, plain.kernels[s], comm.kernels[s])
        seen.add(pol)
    assert seen == {True, False}
    return ulp, l1_rel


def initial_actor_arena(spec, algo, inp):
    return param_arena(build_nets(spec, inp, torch.device(DEV))["policy_net"]).cpu()


def run_pair(case, algo, opt, open_comm, **kw):
    """The same case twice in this process on the same inputs: plain, then through a world-1 communicator.

    The actor's weights after step 0 may differ by 1 ulp (of the weight before the step or after it, whichever is
    larger), except with Adam: its first step normalises the gradient (m / (sqrt(v) + eps) ~ +-1), so a 1-ulp
    change of the gradient moves the update by a few ulps of itself, and where a weight is no larger than the
    lr-sized update that is a few ulps of the weight (4 at most over the cases here)."""
    spec = C.CASES[case] if isinstance(case, str) else case
    p_init = initial_actor_arena(spec, algo, kw.get("inp") or C.make_inputs(spec, algo))
    plain, comm = Recorder(algo), Recorder(algo)
    a = run_cuda_case(case, algo, opt, form="frames", on_step=plain, **kw)
    b = run_cuda_case(case, algo, opt, form="frames", on_step=comm, comm=open_comm, **kw)
    assert engine_of(a["_nets"]).comm is None and engine_of(b["_nets"]).comm is not None
    ulp, l1_rel = check_comm_against_plain(algo, plain, comm, p_init, max_ulp=4.0 if opt == "adam" else 1.0)
    return a, b, ulp, l1_rel


def _pads(res):
    return {"pads": pad_report(res["_nets"], res["_opts"])}


@pytest.mark.parametrize("opt", ["sgd", "sgd_momentum", "adam", "ranger"])
@pytest.mark.parametrize("algo", ["ddpg", "td3"])
@pytest.mark.parametrize("case", ["tiny", "canon"])
def test_step_through_world1_comm(case, algo, opt, open_comm):
    """tiny / canon, 12 steps (policy steps 0 and 10; Ranger's rectification switch and Lookahead at step 6 and
    Lookahead again at 12): bit-identical to the single-GPU step where it must be, and the communicator run against
    the golden fixtures (SGD, Adam: weights, losses and gradients) or the live oracle (SGD with momentum, Ranger)."""
    gold = load_golden("%s_%s_%s.npz" % (algo, case, opt)) if opt in ("sgd", "adam") else None
    inp, dropped = None, 0
    if opt == "sgd_momentum":
        # the seeds are screened for clean ReLU gates along the SGD / Adam / Ranger trajectories only: drop the
        # ambiguous ones of this trajectory from the replayed masks
        inp, dropped, _ = neutralise_ambiguous_gates(C.CASES[case], algo, opt)
    _, b, ulp, l1_rel = run_pair(case, algo, opt, open_comm, golden=gold, inp=inp)
    assert_pads_zero(_pads(b))
    if gold is not None:
        rep = compare_with_golden(b, gold)
        worst = {"loss": max(v for k, v in rep.items() if k.startswith("loss.")),
                 "weight": max(v for k, v in rep.items() if k.startswith("after") and not k.endswith(".delta")),
                 "delta": max(v for k, v in rep.items() if k.endswith(".delta")),
                 "grad": max([v for k, v in rep.items() if k.startswith("grad_")] or [0.0])}
    else:
        inp = inp or C.make_inputs(C.CASES[case], algo)
        # momentum moves the weights up to 1 / (1 - 0.9) times as far as plain SGD, and weights that pass near 0
        # pick up fp32 rounding of about 2 ulp of the tensor's largest weight (canon: 2.2e-5 on this bar, whose floor
        # is 1 such ulp; the bar on the changes, which allows 2 such ulp, is met to 5e-7): the weight bar gets 5e-5,
        # the bar on the changes stays as it is
        worst = assert_oracle_bar(b, run_oracle_case(case, algo, opt, inp=inp), inp["nets"],
                                  rtol=5e-5 if opt == "sgd_momentum" else 1e-5)
        worst["gates_dropped"] = dropped
    print("comm %s %s %s: actor ulp gap after step 0 %.2f, L1 rel gap %.1e, vs oracle %s"
          % (case, algo, opt, ulp, l1_rel, {k: "%.2e" % v for k, v in worst.items()}))


@pytest.mark.parametrize("algo", ["ddpg", "td3"])
@pytest.mark.parametrize("row", SHAPE_ROWS)
def test_step_shapes_rows_through_world1_comm(row, algo, open_comm):
    """The step-shapes rows with SGD (ambiguous ReLU gates dropped): the unfused value head (head gradient from the
    arena, layers 1-2 from partials), action leads 1-3, split-K > 1, H % 4 != 0 and the one-CTA smallest net."""
    spec, inp, dropped, want = prepared(row, algo, "sgd")
    _, b, ulp, l1_rel = run_pair(spec, algo, "sgd", open_comm, inp=inp)
    res = dict({k: v for k, v in b.items() if k.startswith(("final.", "loss."))}, **_pads(b))
    rep = assert_tight_parity(res, want, inp["nets"])
    assert rep["checked"] >= 8, rep
    n_pads = assert_pads_zero(res)
    print("comm %s %s: %d gates dropped, %d pad elements, actor ulp gap %.2f, L1 rel gap %.1e, vs oracle %s"
          % (row, algo, dropped, n_pads, ulp, l1_rel, rep))


@pytest.mark.parametrize("algo", ["ddpg", "td3"])
def test_long_ranger_run_graph_replay_equals_direct(algo, open_comm, monkeypatch):
    """Ranger over 26 steps (policy steps 0, 10 and 20, the last a graph replay; the step counter and the kernel's
    epoch well past a Lookahead cycle): TD3's critics bit-identical to the single-GPU run at every step, and the
    communicator run replayed from CUDA graphs bit-identical to the same run launched directly -- the kernel reads
    its epoch from device memory, so replays must advance it."""
    from recnn_b200.nn.update import _engine
    spec = dict(C.CASES["tiny"], steps=26)
    _, graph, ulp, _ = run_pair(spec, algo, "ranger", open_comm)
    assert engine_of(graph["_nets"]).graphs, "no CUDA graph was captured"
    monkeypatch.setattr(_engine, "_USE_GRAPHS", False)
    direct_rec = Recorder(algo)
    direct = run_cuda_case(spec, algo, "ranger", form="frames", on_step=direct_rec, comm=open_comm)
    assert not engine_of(direct["_nets"]).graphs
    for k in graph:
        if k.startswith(("final.", "loss.")):
            assert np.array_equal(np.asarray(graph[k]).view(np.uint8), np.asarray(direct[k]).view(np.uint8)), k
    for name, o in graph["_opts"].items():
        assert int(o._t[0]) == int(direct["_opts"][name]._t[0]) == (26 if "value" in name else 3), name
        for a in ("_m", "_v", "_slow"):
            assert torch.equal(_bits(getattr(o, a)), _bits(getattr(direct["_opts"][name], a))), (name, a)
    assert_pads_zero(_pads(graph))
    print("comm long %s ranger: actor ulp gap after step 0 %.2f" % (algo, ulp))


# ----------------------------------------------------------------------------- the CUDA-core back end
def simt_worker(in_path, out_path):
    """run_sweep worker: each case plain and through a world-1 communicator, checked against each other here; the
    communicator run's weights, losses and pad report go back for the oracle check."""
    with open(in_path, "rb") as f:
        cases = pickle.load(f)
    out = {}
    for key, (spec, inp) in cases.items():
        row, algo, opt, _ = key
        made = []

        def make(nets):
            made.append(World1Comm(max(param_arena(m).numel() for m in nets.values())))
            return made[-1]

        plain, comm = Recorder(algo), Recorder(algo)
        run_cuda_case(spec, algo, opt, form="frames", inp=inp, on_step=plain)
        b = run_cuda_case(spec, algo, opt, form="frames", inp=inp, on_step=comm, comm=make)
        ulp, l1_rel = check_comm_against_plain(algo, plain, comm, initial_actor_arena(spec, algo, inp))
        out[key] = dict({k: v for k, v in b.items() if k.startswith(("final.", "loss."))}, **_pads(b))
        print("simt comm %s %s: actor ulp gap %.2f, L1 rel gap %.1e" % (row, algo, ulp, l1_rel), file=sys.stderr)
        del b
        gc.collect()
        for c in made:
            c.close()
    with open(out_path, "wb") as f:
        pickle.dump(out, f)


def test_cuda_core_back_end_td3_row(tmp_path):
    """RECNN_B200_MATH=simt: the critics' partials come from the CUDA-core split plan; TD3's critics are again
    bit-identical with and without the communicator, and the communicator run meets the oracle bar."""
    res, err = run_sweep(tmp_path, [(SIMT_ROW, "td3", "sgd", False)], worker="tests.test_comm_world1_gpu:simt_worker",
                         RECNN_B200_MATH="simt")
    print(err[-2000:])
    check_against_oracle(res, "simt-comm")
