"""The DDPG / TD3 update step against the oracle at shapes chosen for the GEMM dispatch edges of step.cu, on both GEMM
back ends, with serialised streams and with the unfused value head; the arena's pad elements; and perf mode (on-device
Philox dropout and TD3 noise) against the oracle fed the host restatement of the device RNG (tests/_philox.py).

Each row of ROWS pins a dispatch edge (S = frame*(dim+1), A = dim, lead = S % 4 zero columns in front of every action
row):
  h50   S 24 (lead 0), A 7,  H 50,  45 rows    H % 4 != 0: tensor-core layer 1 writes an [N, 50] that a CUDA-core
                                                layer 2 reads; unfused value head; odd A < 32
  h96   S 33 (lead 1), A 10, H 96,  130 rows   lead 1; fused head at a non-power-of-2 H; d gen_action on the CUDA cores
  h100  S 102 (lead 2), A 33, H 100, 257 rows  A % 4 = 1 with lead 2 (n_skip, ldA); H % 32 != 0 on the tensor cores
  h320  S 74 (lead 2), A 36, H 320, 1000 rows  H > 256 (unfused, ragged 128-wide tiles); actor dW3 on the tensor cores;
                                                split-K > 1
  h36   S 25 (lead 1), A 4,  H 36,  129 rows   weight_grad with C = 36 (>= 32, % 4 == 0, not % 64)
  h512  S 195 (lead 3), A 64, H 512, 2049 rows lead 3; large H; many splits
  min   S 2 (lead 2),  A 1,  H 3,   2 rows     the smallest legal net
  h64   S 16 (lead 0), A 3,  H 64,  200 rows   lead 0 with H % 4 == 0: d gen_action (the un-gated input gradient) on
                                                the tensor cores; a second fusable H

Ambiguous ReLU gates are removed from the replayed dropout masks (tests/_golden.py:neutralise_ambiguous_gates) and
every weight is held to the golden bar (tests/_golden.py:assert_tight_parity).  The back end, the stream overlap and
the head fusion are read once per process, so those variants run in subprocesses; the CUDA-core and serialised runs
get the oracle's inputs through a pickle and hand their results back the same way."""
from __future__ import annotations

import functools
import os
import pickle
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

import recnn_b200
from recnn_b200.nn.arena import net_layout, param_arena
from oracle import cases as C
from oracle import recnn_oracle as O
from tests import _philox as PH
from tests._cuda import build_nets, build_optimizers, run_cuda_case
from tests._golden import assert_tight_parity, neutralise_ambiguous_gates, oracle_optimizers, run_oracle_case

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# id -> (dim, frame, hidden, n_rows)
ROWS = {"h50": (7, 3, 50, 45), "h96": (10, 3, 96, 130), "h100": (33, 3, 100, 257), "h320": (36, 2, 320, 1000),
        "h36": (4, 5, 36, 129), "h512": (64, 3, 512, 2049), "min": (1, 1, 3, 2), "h64": (3, 4, 64, 200)}
ALGOS = ("ddpg", "td3")
ADAM_ROWS = ("h50", "h320")
RANGER_ROW = "h50"
FUSABLE_ROWS = tuple(r for r, v in ROWS.items() if v[2] % 32 == 0 and 32 <= v[2] <= 256)   # value_head_fusable
SGD_CASES = [(r, a, "sgd", False) for r in ROWS for a in ALGOS]


def row_spec(row, steps=3):
    dim, frame, h, n = ROWS[row]
    i = list(ROWS).index(row)
    return dict(seeds={"ddpg": 4001 + 2 * i, "td3": 4002 + 2 * i}, n_items=3 * n + 50, dim=dim, frame=frame,
                hidden=h, n_rows=n, steps=steps, actor_init_w=6e-1, critic_init_w=54e-2)


@functools.lru_cache(maxsize=None)
def prepared(row, algo, opt):
    """(spec, inputs with the ambiguous gates dropped, units dropped, oracle result)."""
    spec = row_spec(row)
    inp, dropped, _ = neutralise_ambiguous_gates(spec, algo, opt)
    return spec, inp, dropped, run_oracle_case(spec, algo, opt, inp=inp)


# ----------------------------------------------------------------------------- arena pads
def pad_positions(module):
    """Arena indices that hold no parameter: the pitch pads of each weight row and the tails of the bias segments."""
    offs, lds, count = net_layout(module)
    data = np.zeros(count, dtype=bool)
    ps = [module.linear1.weight, module.linear1.bias, module.linear2.weight, module.linear2.bias,
          module.linear3.weight, module.linear3.bias]
    for i, p in enumerate(ps):
        if p.dim() == 2:
            rows, cols = p.shape
            data[(offs[i] + np.arange(rows)[:, None] * lds[i // 2] + np.arange(cols)).reshape(-1)] = True
        else:
            data[offs[i]: offs[i] + p.numel()] = True
    return np.nonzero(~data)[0]


def pad_report(nets, opts):
    """{(net, arena): (pad elements, non-zero pad elements)} over the parameter, gradient and optimizer arenas."""
    owner = {k: k.replace("optimizer", "net") for k in opts}
    by_net = {owner[k]: o for k, o in opts.items()}
    rep = {}
    for name, m in nets.items():
        pos = torch.from_numpy(pad_positions(m)).to(DEV)
        arenas = {"param": param_arena(m), "grad": m.__dict__.get("_recnn_flat_grad")}
        o = by_net.get(name)
        if isinstance(o, recnn_b200.optim._ArenaOptimizer):
            arenas.update(m=o._m, v=o._v, slow=o._slow)
        for k, a in arenas.items():
            if a is not None:
                rep[(name, k)] = (int(pos.numel()), int((a[pos] != 0).sum()))
    return rep


def cuda_result(spec, inp, algo, opt, external):
    got = run_cuda_case(spec, algo, opt, form="frames", inp=inp, external=external)
    nets, opts = got.pop("_nets"), got.pop("_opts")
    res = {k: v for k, v in got.items() if k.startswith(("final.", "loss."))}
    res["pads"] = pad_report(nets, opts)
    return res


def assert_pads_zero(res):
    bad = {k: v for k, v in res["pads"].items() if v[1]}
    assert not bad, "non-zero pad elements (pads, non-zero) per (net, arena): %s" % bad
    return sum(v[0] for v in res["pads"].values())


@functools.lru_cache(maxsize=None)
def default_result(row, algo):
    spec, inp, _, _ = prepared(row, algo, "sgd")
    return cuda_result(spec, inp, algo, "sgd", False)


# ----------------------------------------------------------------------------- subprocess runs
def sweep_worker(in_path, out_path):
    """Entry point of the subprocess runs: the CUDA path on pickled inputs, results pickled back."""
    with open(in_path, "rb") as f:
        cases = pickle.load(f)
    out = {}
    for key, (spec, inp) in cases.items():
        row, algo, opt, external = key
        print("[case] %s %s %s %s" % key, file=sys.stderr, flush=True)
        out[key] = cuda_result(spec, inp, algo, opt, external)
    with open(out_path, "wb") as f:
        pickle.dump(out, f)


def run_sweep(tmp_path, keys, worker="tests.test_step_shapes_gpu:sweep_worker", **env):
    """Run the CUDA side of ``keys`` in a fresh process with ``env`` set; returns (results, stderr).  ``worker``:
    "module:function" taking (inputs pickle, results pickle), sweep_worker's contract."""
    cases = {k: prepared(*k[:3])[:2] for k in keys}
    in_path, out_path = str(tmp_path / "cases.pkl"), str(tmp_path / "results.pkl")
    with open(in_path, "wb") as f:
        pickle.dump(cases, f)
    mod, fn = worker.split(":")
    code = ("import sys, importlib; sys.path.insert(0, %r); importlib.import_module(%r).%s(%r, %r)"
            % (ROOT, mod, fn, in_path, out_path))
    e = dict(os.environ)
    for k in ("RECNN_B200_MATH", "RECNN_B200_OVERLAP", "RECNN_B200_FUSE_HEAD", "RECNN_B200_DEBUG", "RECNN_B200_GRAPHS"):
        e.pop(k, None)
    e.update(env)
    r = subprocess.run([sys.executable, "-c", code], env=e, capture_output=True, text=True, cwd=ROOT)
    assert r.returncode == 0, (r.stdout[-3000:], r.stderr[-3000:])
    with open(out_path, "rb") as f:
        return pickle.load(f), r.stderr


def check_against_oracle(results, label):
    worst = {"loss": 0.0, "weight": 0.0, "delta": 0.0}
    for key, res in results.items():
        row, algo, opt, _ = key
        _, inp, dropped, want = prepared(row, algo, opt)
        rep = assert_tight_parity(res, want, inp["nets"])
        assert rep["checked"] >= 8, (key, rep)
        assert_pads_zero(res)
        for k in worst:
            worst[k] = max(worst[k], rep[k])
        print("%s %s: %d gates dropped, max err loss %.2e weight %.2e delta %.2e"
              % (label, key, dropped, rep["loss"], rep["weight"], rep["delta"]))
    print("%s worst: %s" % (label, worst))


# ----------------------------------------------------------------------------- default back end, in process
@pytest.mark.parametrize("algo", ALGOS)
@pytest.mark.parametrize("row", list(ROWS))
def test_step_shapes_vs_oracle(row, algo):
    """SGD(1e-3), three steps from a policy step: the tight bar on every weight, and every pad element still 0."""
    _, inp, dropped, want = prepared(row, algo, "sgd")
    res = default_result(row, algo)
    rep = assert_tight_parity(res, want, inp["nets"])
    n_pads = assert_pads_zero(res)
    print("%s %s: %d gates dropped, %d pad elements, %s" % (row, algo, dropped, n_pads, rep))
    assert rep["checked"] >= 8, rep


def test_rows_have_pads_and_lead_columns():
    """The matrix does exercise what it is meant to: pitch pads and bias tails, every lead value, A % 4 != 0."""
    leads = {(f * (d + 1)) % 4 for d, f, _, _ in ROWS.values()}
    assert leads == {0, 1, 2, 3}
    assert any(d % 4 for d, _, _, _ in ROWS.values()) and any(h % 4 for _, _, h, _ in ROWS.values())
    assert FUSABLE_ROWS and any(h > 256 for _, _, h, _ in ROWS.values())


@pytest.mark.parametrize("external", [False, True], ids=["builtin", "torch"])
@pytest.mark.parametrize("algo", ALGOS)
@pytest.mark.parametrize("row", ADAM_ROWS)
def test_step_shapes_adam(row, algo, external):
    """Adam(1e-5): the built-in optimizer reads layers 1-2 straight from the split-K partials (GradSource); an external
    torch.optim.Adam cuts the step into phases around optimizer.step().  Both meet the same bar."""
    spec, inp, dropped, want = prepared(row, algo, "adam")
    res = cuda_result(spec, inp, algo, "adam", external)
    # Adam's g / (|g| + eps) turns the fp32 rounding of a gradient that nearly cancels into an lr-sized difference of
    # that element (at h320 a few of the 100k-element critic weights, on the built-in and the torch optimizer alike).
    # A handful per tensor may miss the bar, each by at most the 3 steps' worth of lr = 1e-5 it can move.
    rep = assert_tight_parity(res, want, inp["nets"], outliers=8, outlier_abs=2 * 3 * 1e-5)
    assert_pads_zero(res)
    print("%s %s adam external=%s: %d gates dropped, %s" % (row, algo, external, dropped, rep))


@pytest.mark.parametrize("algo", ALGOS)
def test_ranger_keeps_pads_zero(algo):
    """Ranger's moment and slow-weight arenas have the parameter arena's geometry: their pads stay 0 as well."""
    spec, inp, dropped, want = prepared(RANGER_ROW, algo, "ranger")
    res = cuda_result(spec, inp, algo, "ranger", False)
    assert any(k[1] == "slow" and v[0] > 0 for k, v in res["pads"].items())
    assert_pads_zero(res)
    rep = assert_tight_parity(res, want, inp["nets"])
    print("%s %s ranger: %d gates dropped, %s" % (RANGER_ROW, algo, dropped, rep))


# ----------------------------------------------------------------------------- other back ends / switches
def test_step_shapes_on_the_cuda_core_back_end(tmp_path):
    """RECNN_B200_MATH=simt: every contraction on the exact-fp32 CUDA-core kernel, the same bar."""
    res, _ = run_sweep(tmp_path, SGD_CASES, RECNN_B200_MATH="simt")
    check_against_oracle(res, "simt")


def test_serialised_streams_are_bit_identical(tmp_path):
    """RECNN_B200_OVERLAP=0 issues the same kernels in the same reduction orders on one stream: the final weights and
    losses are bit-identical to the default (three-stream) run."""
    res, _ = run_sweep(tmp_path, SGD_CASES, RECNN_B200_OVERLAP="0")
    for key, r in res.items():
        d = default_result(key[0], key[1])
        for k in d:
            if k.startswith(("final.", "loss.")):
                assert np.array_equal(np.asarray(r[k]).view(np.uint8), np.asarray(d[k]).view(np.uint8)), (key, k)


def test_unfused_value_head(tmp_path):
    """RECNN_B200_FUSE_HEAD=0 on the rows whose H the fused value-head kernel takes: head kernel, head-gradient
    partials and their reduction instead, the same bar."""
    res, _ = run_sweep(tmp_path, [(r, a, "sgd", False) for r in FUSABLE_ROWS for a in ALGOS], RECNN_B200_FUSE_HEAD="0")
    check_against_oracle(res, "unfused-head")


EPI_NAMES = {0: "HIDDEN", 1: "LINEAR", 2: "GATE", 3: "STORE", 4: "PARTIAL", 5: "ACCUM"}
# the tensor-core variants (EPI, A_MN, B_MN) the DDPG / TD3 step issues: gemm_nt (hidden layers, output layers),
# backprop_hidden (gated / plain input gradients) and weight_grad (split-K partials)
STEP_TC_VARIANTS = {("HIDDEN", 0, 0), ("LINEAR", 0, 0), ("GATE", 0, 1), ("STORE", 0, 1), ("PARTIAL", 1, 1)}
_TC_LINE = re.compile(r"^\[tc_gemm\] BN=(\d+) A_MN=(\d) B_MN=(\d) EPI=(\d) M=(\d+) N=(\d+) K0=(\d+) K1=(\d+)")


def parse_tc_launches(stderr):
    """{case key: [(EPI, A_MN, B_MN, BN, M, N, K0, K1)]} from a RECNN_B200_DEBUG=1 run of sweep_worker."""
    per, cur = {}, None
    for line in stderr.splitlines():
        if line.startswith("[case] "):
            cur = tuple(line.split()[1:3])
            per.setdefault(cur, [])
            continue
        m = _TC_LINE.match(line)
        if m:
            bn, amn, bmn, epi, M, N, K0, K1 = (int(x) for x in m.groups())
            per[cur].append((EPI_NAMES[epi], amn, bmn, bn, M, N, K0, K1))
    return per


@pytest.mark.parametrize("math", ["default", "simt"])
def test_backend_coverage_from_debug_log(tmp_path, math):
    """RECNN_B200_DEBUG=1 logs every tensor-core launch (and synchronises after it, so graphs are off).  The default
    back end must launch every tensor-core variant the step can reach over the sweep; RECNN_B200_MATH=simt none."""
    env = dict(RECNN_B200_DEBUG="1", RECNN_B200_GRAPHS="0")
    if math == "simt":
        env["RECNN_B200_MATH"] = "simt"
    _, err = run_sweep(tmp_path, SGD_CASES, **env)
    assert "[tc_gemm] FAILED" not in err
    per = parse_tc_launches(err)
    assert set(per) == {(r, a) for r in ROWS for a in ALGOS}
    if math == "simt":
        assert not any(per.values()), {k: v[:3] for k, v in per.items() if v}
        return
    for key, launches in sorted(per.items()):
        kinds = {}
        for epi, amn, bmn, bn, M, N, K0, K1 in launches:
            kinds.setdefault("%s(%d%d)" % (epi, amn, bmn), set()).add((M, N, K0, K1, bn))
        print(key, {k: sorted(v) for k, v in sorted(kinds.items())})
    seen = {(epi, amn, bmn) for v in per.values() for epi, amn, bmn, *_ in v}
    assert seen == STEP_TC_VARIANTS, seen
    assert {bn for v in per.values() for _, _, _, bn, *_ in v} == {64, 128}
    # H % 4 != 0 keeps every hidden-to-hidden GEMM off the tensor cores; the smallest net only has room for layer 1
    for key, launches in per.items():
        H = ROWS[key[0]][2]
        if H % 4:
            assert not any(epi == "HIDDEN" and K0 == H for epi, _, _, _, _, _, K0, _ in launches), key


# ----------------------------------------------------------------------------- perf mode
# (dim, frame, hidden, n_rows, torch seed): H a multiple of 32, and H = 100 (keep bits straddle 32-bit words).  The
# seeds give oracle runs with no kept pre-activation within C.GATE_GUARD of 0 over the three steps (asserted below).
PERF_SHAPES = {"p64": (10, 3, 64, 120, {"ddpg": 1, "td3": 1}), "p100": (33, 3, 100, 100, {"ddpg": 3, "td3": 3})}
PERF_STEPS = (0, 10, 20)     # three policy steps: the first runs directly, the next two replay one CUDA graph


def perf_spec(shape, algo):
    dim, frame, h, n, _ = PERF_SHAPES[shape]
    return dict(seeds={"ddpg": 77, "td3": 78}, n_items=2 * n + 40, dim=dim, frame=frame, hidden=h, n_rows=n,
                steps=len(PERF_STEPS), actor_init_w=6e-1, critic_init_w=54e-2)


def perf_oracle(shape, algo, seed):
    """The oracle fed the host restatement of the masks / noise of rng steps 0, 1, 2; returns (want, inputs, gate log)."""
    spec = perf_spec(shape, algo)
    inp = C.make_inputs(spec, algo)
    n, H, A = spec["n_rows"], spec["hidden"], spec["dim"]
    nets = {k: O.copy_net(v) for k, v in inp["nets"].items()}
    opts = oracle_optimizers("sgd", algo)
    batch = O.frame_gather(inp["table"], inp["items"], inp["ratings"], inp["sizes"], spec["frame"])
    params = dict(C.DDPG_PARAMS if algo == "ddpg" else C.TD3_PARAMS)
    losses = {}
    O.GATE_LOG.update(on=True, thresh=float(C.GATE_GUARD), hits=[])
    try:
        for k, step in enumerate(PERF_STEPS):
            masks = PH.step_masks(seed, k, n, H, algo)
            if algo == "ddpg":
                loss, _ = O.ddpg_update(batch, params, nets, opts, masks, step)
            else:
                noise = PH.td3_noise(seed, k, n, A, params["noise_std"]).astype(np.float32)
                loss, _ = O.td3_update(batch, params, nets, opts, masks, noise, step)
            for key, v in loss.items():
                if key != "step":
                    losses.setdefault("loss." + key, []).append(v)
    finally:
        O.GATE_LOG["on"] = False
    hits, O.GATE_LOG["hits"] = O.GATE_LOG["hits"], []
    want = {k: np.asarray(v, dtype=np.float64) for k, v in losses.items()}
    for name, p in nets.items():
        for t, v in p.items():
            want["final.%s.%s" % (name, t)] = v
    return want, inp, sum(int(r.size) for _, r, _ in hits)


def _frames_batch(spec, inp):
    return {"items": torch.from_numpy(inp["items"]), "ratings": torch.from_numpy(inp["ratings"]),
            "sizes": torch.from_numpy(inp["sizes"]), "table": torch.from_numpy(inp["table"]).to(DEV)}


def check_perf_steps(shape, algo):
    """Three perf-mode steps (no masks, no noise passed) against the oracle fed the host masks of rng steps 0, 1, 2
    (and the host noise): the tight bar.  A wrong keep bit, stream, straddle, noise transform or an rng_step that
    does not advance through graph replays moves whole rows of the gradients."""
    seed = PERF_SHAPES[shape][4][algo]
    want, inp, ambiguous = perf_oracle(shape, algo, seed)
    assert ambiguous == 0, "seed %d has %d ambiguous gates: pick another" % (seed, ambiguous)
    spec = perf_spec(shape, algo)
    dev = torch.device(DEV)
    torch.manual_seed(seed)                  # the engine keys Philox on torch.initial_seed() when it is created
    nets = build_nets(spec, inp, dev)
    opts = build_optimizers("sgd", nets, algo)
    params = dict(C.DDPG_PARAMS if algo == "ddpg" else C.TD3_PARAMS)
    update = recnn_b200.nn.ddpg_update if algo == "ddpg" else recnn_b200.nn.td3_update
    got = {}
    batch = _frames_batch(spec, inp)
    for step in PERF_STEPS:
        loss = update(dict(batch), params, nets, opts, dev, {}, recnn_b200.utils.DummyWriter(), learn=True, step=step)
        for k, v in loss.items():
            if k != "step":
                got.setdefault("loss." + k, []).append(v)
    got = {k: np.asarray(v, dtype=np.float64) for k, v in got.items()}
    from tests._cuda import dump_net
    for name, m in nets.items():
        for t, v in dump_net(m).items():
            got["final.%s.%s" % (name, t)] = v
    rep = assert_tight_parity(got, want, inp["nets"])
    print("perf %s %s seed %d: %s" % (shape, algo, seed, rep))


def check_perf_forward(shape, algo):
    """One train-mode step with learn=False: gen_action is the oracle actor on the host keep masks of the policy's
    streams at rng step 0; TD3's next_action is the eval target actor plus the clipped host noise of stream 15."""
    seed = PERF_SHAPES[shape][4][algo]
    spec = perf_spec(shape, algo)
    inp = C.make_inputs(spec, algo)
    n, H, A = spec["n_rows"], spec["hidden"], spec["dim"]
    dev = torch.device(DEV)
    torch.manual_seed(seed)
    nets = build_nets(spec, inp, dev)
    params = dict(C.DDPG_PARAMS if algo == "ddpg" else C.TD3_PARAMS)
    ref = O.frame_gather(inp["table"], inp["items"], inp["ratings"], inp["sizes"], spec["frame"])
    batch = {k: torch.from_numpy(v) for k, v in ref.items()}
    opts = {k: None for k in (("policy_optimizer", "value_optimizer") if algo == "ddpg" else
                              ("policy_optimizer", "value_optimizer1", "value_optimizer2"))}
    update = recnn_b200.nn.ddpg_update if algo == "ddpg" else recnn_b200.nn.td3_update
    debug = {}
    update(batch, params, nets, opts, dev, debug, recnn_b200.utils.DummyWriter(), learn=False, step=0)
    assert set(debug) >= {"gen_action", "next_action"}
    s0, s1 = (PH.DDPG_STREAMS if algo == "ddpg" else PH.TD3_STREAMS)["policy"]
    want_gen, _ = O.actor_forward(inp["nets"]["policy_net"], ref["state"].astype(np.float64),
                                  (PH.keep_mask(seed, 0, s0, n, H), PH.keep_mask(seed, 0, s1, n, H)))
    got_gen = debug["gen_action"].cpu().numpy().astype(np.float64)
    scale = np.abs(want_gen).max()
    err = float(np.max(np.abs(got_gen - want_gen)))
    assert err <= 1e-5 * scale, (err, scale)
    # the eval-mode forward draws no masks: the train-mode one must differ from it
    eval_gen, _ = O.actor_forward(inp["nets"]["policy_net"], ref["state"].astype(np.float64))
    assert np.max(np.abs(got_gen - eval_gen)) > 1e-2 * scale
    want_next, _ = O.actor_forward(inp["nets"]["target_policy_net"], ref["next_state"].astype(np.float64))
    if algo == "td3":
        clip = params["noise_clip"]
        want_next = want_next + np.clip(PH.td3_noise(seed, 0, n, A, params["noise_std"]), -clip, clip)
    got_next = debug["next_action"].cpu().numpy().astype(np.float64)
    scale_n = np.abs(want_next).max()
    err_n = float(np.max(np.abs(got_next - want_next)))
    assert err_n <= 1e-5 * scale_n, (err_n, scale_n)
    print("perf forward %s %s: gen %.2e, next %.2e of max" % (shape, algo, err / scale, err_n / scale_n))


@pytest.mark.parametrize("algo", ALGOS)
@pytest.mark.parametrize("shape", list(PERF_SHAPES))
def test_perf_mode_forward_draws_documented_bits(shape, algo):
    check_perf_forward(shape, algo)


@pytest.mark.parametrize("algo", ALGOS)
@pytest.mark.parametrize("shape", list(PERF_SHAPES))
def test_perf_mode_steps_vs_oracle(shape, algo):
    check_perf_steps(shape, algo)


def test_perf_mode_on_the_cuda_core_back_end():
    """The same perf-mode checks with every GEMM on the CUDA cores: both epilogues draw the same bits."""
    calls = "; ".join("T.check_perf_forward(%r, %r); T.check_perf_steps(%r, %r)" % (s, a, s, a)
                      for s in PERF_SHAPES for a in ALGOS)
    code = "import sys; sys.path.insert(0, %r); from tests import test_step_shapes_gpu as T; %s" % (ROOT, calls)
    env = dict(os.environ, RECNN_B200_MATH="simt")
    r = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, cwd=ROOT)
    print(r.stdout[-3000:], r.stderr[-3000:])
    assert r.returncode == 0
