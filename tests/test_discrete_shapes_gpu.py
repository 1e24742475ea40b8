"""The REINFORCE policy gradient, the item-id critic step and the Beta step against their float64 / one-hot oracles at
the shapes of tests/_discrete_shapes.py:ROWS, each row chosen for a dispatch edge of the contraction helpers they share
with the DDPG step (gemm_nt, linear_out, backprop_hidden, weight_grad) and of their own chunk-width GEMMs.  The sweep
runs on the default back end in process, then in subprocesses (the back end is read once per process) on the CUDA-core
back end and with the tensor-core launch log on, whose lines show which back end each GEMM took."""
from __future__ import annotations

import functools
import os
import pickle
import re
import subprocess
import sys
import time

import numpy as np
import pytest
import torch

import recnn_b200
from recnn_b200.nn import beta as BM
from recnn_b200.nn.update import reinforce as RF
from oracle import cases as C
from oracle import recnn_oracle as O
from oracle import reinforce_oracle as RO
from tests import _discrete_shapes as D
from tests._cuda import dump_grad, dump_net, load_net
from tests._discrete import make_policy
from tests._golden import assert_tight_parity
from tests.test_reinforce_chunked_gpu import REORDER_BAR, policy_grad

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ROWS = list(D.ROWS)
KEYS = ([("pg", r, m, K) for r in ROWS for m, K in D.PG_CASES] + [("critic", r, t) for r in ROWS for t in (0, 1)]
        + [("beta", r) for r in ROWS])


@pytest.fixture(scope="module", autouse=True)
def wall_time():
    t0 = time.time()
    yield
    print("\n%s: wall time %.1f s" % (os.path.basename(__file__), time.time() - t0))


# ----------------------------------------------------------------------------- inputs and oracles (host)
@functools.lru_cache(maxsize=None)
def inputs(key):
    if key[0] == "pg":
        return D.pg_inputs(key[1])
    if key[0] == "critic":
        return D.critic_inputs(key[1], bool(key[2]))
    return D.beta_inputs(key[1])


@functools.lru_cache(maxsize=None)
def critic_grads(key):
    return D.critic_grads_f64(inputs(key), D.dims(key[1])["I"])


@functools.lru_cache(maxsize=None)
def oracle(key):
    inp = inputs(key)
    if key[0] == "pg":
        return D.pg_oracle(inp, key[2], key[3])
    if key[0] == "critic":
        return D.critic_oracle(inp, D.dims(key[1])["I"])
    return D.beta_oracle(inp)


# ----------------------------------------------------------------------------- the CUDA side
def _np(t):
    return t.detach().double().cpu().numpy()


def cuda_pg(key, inp):
    """recnn_reinforce_policy_grad_chunked at the row's chunk width and as one chunk; on the peaked row also over the
    clamped rows alone."""
    _, row, method, K = key
    d = D.dims(row)
    mid = RO.METHODS[method]
    m = make_policy(inp["p"], d["S"], d["H"], d["I"])
    t = {k: torch.from_numpy(np.ascontiguousarray(inp[k])).to(DEV) for k in ("state", "action", "blp", "ret")}

    def call(rows, chunk):
        loss, oob, g = policy_grad(m, t["state"][rows].contiguous(), t["action"][rows].contiguous(),
                                   None if mid == RO.BASIC else t["blp"][rows].contiguous(),
                                   t["ret"][rows].contiguous(), mid, K, chunk)
        return loss, oob, {k: _np(v) for k, v in g.items()}

    everything = torch.arange(d["n"], device=DEV)
    out = {"chunked": call(everything, d["chunk"] if d["chunk"] < d["I"] else d["I"]),
           "single": call(everything, d["I"])}
    if row == D.PEAK_ROW:
        clamped = np.nonzero(D.clamp_classes(inp) != 0)[0]
        out["clamped"] = call(torch.from_numpy(clamped).to(DEV), d["chunk"])
    return out


def cuda_critic(key, inp):
    """CRITIC_STEPS Adam steps of value_update with item ids (chunk width forced) and with the dense one-hot; then the
    gradient of each of D.grad_batches at the initial weights on both paths, read from .grad under an external SGD at
    lr 0 (which leaves the weights where they are)."""
    _, row, train = key
    d = D.dims(row)
    S, H, Hp, I = d["S"], d["H"], d["Hp"], d["I"]

    def agent(sgd=False):
        algo = recnn_b200.nn.Reinforce(make_policy(inp["pp"], S, Hp, I), load_net(recnn_b200.nn.Critic(S, I, H, 0.3),
                                                                                   inp["cp"], DEV))
        algo.nets["value_net"].train(bool(train))
        params = algo.nets["value_net"].parameters()
        algo.optimizers["value_optimizer"] = (torch.optim.SGD(params, lr=0.0) if sgd
                                              else recnn_b200.optim.Adam(params, lr=D.LR))
        return algo

    ids_algo, dense_algo = agent(), agent()
    params = dict(ids_algo.params, **D.CRITIC_PARAMS)
    to = lambda bb: {k: torch.from_numpy(v) for k, v in bb.items()}                     # noqa: E731
    saved = RF._chunk_items
    RF._chunk_items = lambda n, items: min(d["chunk"], items)
    try:
        got, dense = [], []
        for step, (b, masks) in enumerate(zip(inp["batches"], inp["masks"])):
            extra = {} if masks is None else {"dropout_masks": [torch.from_numpy(m) for m in masks * 3]}
            got.append(float(recnn_b200.nn.value_update({**to(b), **extra}, params, ids_algo.nets,
                                                         ids_algo.optimizers, torch.device(DEV), {}, learn=True,
                                                         step=step)))
            dense.append(float(recnn_b200.nn.value_update({**to(D.one_hot(b, I)), **extra}, params, dense_algo.nets,
                                                           dense_algo.optimizers, torch.device(DEV), {}, learn=True,
                                                           step=step)))
        grads = []
        ids_sgd, dense_sgd = agent(True), agent(True)
        for b, masks in D.grad_batches(inp, I):
            extra = {} if masks is None else {"dropout_masks": [torch.from_numpy(m) for m in masks * 3]}
            one = []
            for algo, batch in ((ids_sgd, b), (dense_sgd, D.one_hot(b, I))):
                loss = recnn_b200.nn.value_update({**to(batch), **extra}, params, algo.nets, algo.optimizers,
                                                  torch.device(DEV), {}, learn=True)
                one.append((float(loss), dump_grad(algo.nets["value_net"])))
            grads.append(one)
    finally:
        RF._chunk_items = saved
    return {"loss": np.asarray(got), "dense_loss": np.asarray(dense), "final": dump_net(ids_algo.nets["value_net"]),
            "dense_final": dump_net(dense_algo.nets["value_net"]), "grads": grads}


def cuda_beta(key, inp):
    """BETA_CALLS calls of Beta.forward (recnn_beta_step, built-in RAdam) at the row's chunk width."""
    d = D.dims(key[1])
    beta = recnn_b200.nn.Beta(d["S"], d["I"])
    beta.load_state_dict({"net.0.weight": torch.from_numpy(inp["w"]), "net.0.bias": torch.from_numpy(inp["b"])})
    beta = beta.to(DEV)
    saved = BM._chunk_items
    BM._chunk_items = lambda rows, items: min(d["chunk"], items)
    try:
        out = {"probs": [], "loss": [], "gw": [], "gb": []}
        for s, ids in inp["calls"]:
            p = beta(torch.from_numpy(s).to(DEV), torch.from_numpy(ids).to(DEV))
            out["probs"].append(_np(p))
            out["loss"].append(float(beta.last_loss))
            out["gw"].append(_np(beta.net[0].weight.grad))
            out["gb"].append(_np(beta.net[0].bias.grad))
    finally:
        BM._chunk_items = saved
    out["w"] = beta.net[0].weight.detach().cpu().numpy().copy()
    out["b"] = beta.net[0].bias.detach().cpu().numpy().copy()
    return out


RUN = {"pg": cuda_pg, "critic": cuda_critic, "beta": cuda_beta}


def run_case(key, inp):
    return RUN[key[0]](key, inp)


# ----------------------------------------------------------------------------- the checks
def _rel(got, want):
    scale = float(np.abs(want).max())
    err = float(np.abs(got - want).max())
    return err / scale if scale > 0 else (0.0 if err == 0 else float("inf"))


def check_pg(key, res):
    """The bars of test_reinforce_chunked_gpu.py: loss rel 2e-4, every gradient within 3e-4 of its largest element;
    chunked vs one chunk within REORDER_BAR; every gradient entry written."""
    want_loss, want, aux = oracle(key)
    loss, oob, got = res["chunked"]
    rep = {"loss": abs(loss - want_loss) / abs(want_loss)}
    classes = D.clamp_classes(inputs(key))
    assert not (classes == 2).any(), key          # no pi(a) so close to eps or 1 - eps that fp32 cannot place it
    assert oob == 0, key
    assert loss == pytest.approx(want_loss, rel=2e-4, abs=1e-4 * (1 + abs(want_loss))), key
    for k in ("w1", "b1", "w2", "b2"):
        assert np.isfinite(got[k]).all(), (key, k)
        rep[k] = _rel(got[k], want[k])
        assert rep[k] <= 3e-4, (key, k, rep)
    l1, oob1, single = res["single"]
    assert oob1 == 0
    # test_reinforce_chunked_gpu.py holds the reordered loss to rel 1e-5 at 40 rows and to 1e-6 of the sum of |row
    # terms| at 4096 rows: the loss is a sum of signed terms that can cancel (at 1000 rows to 1e-4 of that sum)
    abs_sum = float(np.abs(aux["row_loss"]).sum())
    rep["loss_reorder"] = abs(loss - l1) / abs_sum
    assert loss == pytest.approx(l1, rel=1e-5, abs=1e-6) or abs(loss - l1) <= 1e-6 * abs_sum, (key, loss, l1, abs_sum)
    rep["reorder"] = max(_rel(got[k], single[k]) for k in single)
    assert rep["reorder"] <= REORDER_BAR, (key, rep)
    if "clamped" in res:
        assert (classes == 1).any() and (classes == -1).any() and (classes == 0).any()
        rows = classes != 0
        lc, oobc, gc = res["clamped"]
        assert oobc == 0
        for k, v in gc.items():          # pi(a) outside [eps, 1 - eps]: the clamp's zero slope, exactly
            assert not np.any(v), (key, k)
        want_c = float(aux["row_loss"][rows].sum())
        assert lc == pytest.approx(want_c, rel=2e-4, abs=1e-4 * (1 + abs(want_c))), (key, lc, want_c)
        rep["clamped_rows"] = int(rows.sum())
    return rep


def _blocks(g, S):
    """A critic gradient with layer 1 split into its state block and its action block."""
    out = {k: v for k, v in g.items() if k != "w1"}
    out["w1.state"], out["w1.action"] = g["w1"][:, :S], g["w1"][:, S:]
    return out


def check_critic(key, res):
    """The gradient of every batch pattern (all rows on one id, distinct ids, ids of the last chunk) at the initial
    weights against float64 autograd: each tensor within 1e-4 of its largest element on both paths, unselected action
    columns exactly 0 on the item-id path (test_action_block_gradient_structure_and_determinism's bars).  Then three
    Adam steps with the bars of test_ids_match_oracle_and_dense_path."""
    _, row, train = key
    d = D.dims(row)
    S, I = d["S"], d["I"]
    rep = {"grad": 0.0, "grad_dense": 0.0, "grad_vs_dense": 0.0}
    for (b, _), want, got in zip(D.grad_batches(inputs(key), I), critic_grads(key), res["grads"]):
        want_l, want_g = want[0], _blocks(want[1], S)
        (l_ids, g_ids), (l_dense, g_dense) = got
        assert l_ids == pytest.approx(want_l, rel=2e-5, abs=1e-6), (key, l_ids, want_l)
        assert l_dense == pytest.approx(want_l, rel=2e-5, abs=1e-6), (key, l_dense, want_l)
        g_ids, g_dense = _blocks(g_ids, S), _blocks(g_dense, S)
        for t, w in want_g.items():
            e_ids, e_dense = _rel(g_ids[t], w), _rel(g_dense[t], w)
            rep["grad"], rep["grad_dense"] = max(rep["grad"], e_ids), max(rep["grad_dense"], e_dense)
            rep["grad_vs_dense"] = max(rep["grad_vs_dense"], _rel(g_ids[t], g_dense[t]))
            assert e_ids <= 1e-4 and e_dense <= 1e-4, (key, t, e_ids, e_dense)
        unselected = np.ones(I, bool)
        unselected[b["action"]] = False
        assert not np.any(g_ids["w1.action"][:, unselected]), key
    want_loss, want_net, margin = oracle(key)
    assert margin > C.GATE_GUARD, (key, margin)
    rep["loss"] = float(np.max(np.abs(res["loss"] - want_loss) / np.abs(want_loss)))
    for g, dn, w in zip(res["loss"], res["dense_loss"], want_loss):
        assert g == pytest.approx(w, rel=2e-5, abs=1e-6), (key, res["loss"], want_loss)
        assert g == pytest.approx(dn, rel=1e-5, abs=1e-7), (key, res["loss"], res["dense_loss"])
    # One chunk: that test's single-chunk bars on every element.  Several chunks: its forced-chunk bar,
    # 1e-4 |w| + 1e-5 max |w|, on every element but at most 2 per tensor, each within the 2 * steps * lr that Adam's
    # g / (|g| + eps) can move an element whose gradient nearly cancels (on the dense CUDA path as on the item-id one).
    single = d["chunk"] >= I
    rep["outliers"] = 0
    rep["weight"] = rep["vs_dense"] = 0.0
    for t in O.PARAM_ORDER:
        w, got, dense = want_net[t], res["final"][t], res["dense_final"][t]
        scale = np.abs(w).max()
        rep["vs_dense"] = max(rep["vs_dense"], float(np.abs(got - dense).max() / scale))
        if single:
            np.testing.assert_allclose(got, w, rtol=1e-4, atol=1e-5 * scale, err_msg="%s %s" % (key, t))
            assert np.abs(got - dense).max() <= 2e-6 * scale, (key, t)
        bar = 1e-4 * np.abs(w) + 1e-5 * scale
        for other in (w, dense):
            off = np.abs(got - other) > bar
            rep["outliers"] = max(rep["outliers"], int(off.sum()))
            assert off.sum() <= 2, (key, t, int(off.sum()))
            assert not off.any() or np.abs(got - other)[off].max() <= 2 * D.CRITIC_STEPS * D.LR, (key, t)
        ok = np.abs(got - w) <= bar
        rep["weight"] = max(rep["weight"], float(np.max(np.abs(got - w)[ok] / (np.abs(w)[ok] + 0.1 * scale))))
    return rep


def check_beta(key, res):
    """The bars of test_beta_gpu.py::oracle_sweep_case."""
    inp = inputs(key)
    want_p, want_l, want_g, want_params = oracle(key)
    rep = {"probs": 0.0, "loss": 0.0, "grad_w": 0.0, "grad_b": 0.0}
    for t in range(D.BETA_CALLS):
        p, wp = res["probs"][t], want_p[t]
        rep["probs"] = max(rep["probs"], float(np.max(np.abs(p - wp) / (wp + 1e-2 * wp.max()))))
        rep["loss"] = max(rep["loss"], abs(res["loss"][t] - want_l[t]) / (abs(want_l[t]) + 0.1))
        rep["grad_w"] = max(rep["grad_w"], _rel(res["gw"][t], want_g[t]["w"]))
        rep["grad_b"] = max(rep["grad_b"], _rel(res["gb"][t], want_g[t]["b"]))
    assert rep["probs"] <= 1e-5 and rep["loss"] <= 1e-5, (key, rep)
    assert rep["grad_w"] <= 1e-4 and rep["grad_b"] <= 1e-4, (key, rep)
    tight = assert_tight_parity({"final.beta.w": res["w"], "final.beta.b": res["b"]},
                                {"final.beta.w": want_params["w"], "final.beta.b": want_params["b"]},
                                {"beta": {"w": inp["w"], "b": inp["b"]}})
    rep["weight"] = tight["weight"]
    return rep


CHECK = {"pg": check_pg, "critic": check_critic, "beta": check_beta}


def check(key, res, label):
    rep = CHECK[key[0]](key, res)
    print("%s %s: %s" % (label, " ".join(map(str, key)), " ".join("%s %.2e" % kv if isinstance(kv[1], float)
                                                                 else "%s %s" % kv for kv in rep.items())))
    return rep


# the quantity of each section summarised per row: the worst gradient of the policy against float64, the worst
# critic gradient against float64 (both paths), the worst Beta probability and gradient
ROW_SUMMARY = {"pg": ("w1", "b1", "w2", "b2"), "critic": ("grad", "grad_dense"), "beta": ("probs", "grad_w", "grad_b")}


def check_all(results, label):
    worst, per_row = {}, {}
    for key in KEYS:
        rep = check(key, results[key], label)
        for k, v in rep.items():
            if isinstance(v, float):
                worst[(key[0], k)] = max(worst.get((key[0], k), 0.0), v)
                if k in ROW_SUMMARY[key[0]]:
                    per_row[(key[1], key[0])] = max(per_row.get((key[1], key[0]), 0.0), v)
    for row in ROWS:
        print("%s worst, row %s: %s" % (label, row, "  ".join("%s %.1e" % (sec, per_row[(row, sec)])
                                                                 for sec in ROW_SUMMARY)))
    print("%s worst: %s" % (label, {"%s.%s" % k: "%.2e" % v for k, v in sorted(worst.items())}))


# ----------------------------------------------------------------------------- default back end, in process
@pytest.mark.parametrize("row", ROWS)
def test_policy_gradient_vs_float64(row):
    for key in (k for k in KEYS if k[0] == "pg" and k[1] == row):
        assert D.pg_margin(inputs(key)) > C.GATE_GUARD, key
        check(key, run_case(key, inputs(key)), "default")


@pytest.mark.parametrize("train", [0, 1], ids=["eval", "train"])
@pytest.mark.parametrize("row", ROWS)
def test_item_id_critic_vs_one_hot_oracle(row, train):
    key = ("critic", row, train)
    check(key, run_case(key, inputs(key)), "default")


@pytest.mark.parametrize("row", ROWS)
def test_beta_vs_float64(row):
    key = ("beta", row)
    check(key, run_case(key, inputs(key)), "default")


# ----------------------------------------------------------------------------- subprocess runs
def sweep_worker(in_path, out_path):
    """Entry point of the subprocess runs: every key on its pickled inputs, results pickled back."""
    with open(in_path, "rb") as f:
        cases = pickle.load(f)
    out = {}
    for key, inp in cases.items():
        print("[case] %s" % " ".join(map(str, key)), file=sys.stderr, flush=True)
        out[key] = run_case(key, inp)
    with open(out_path, "wb") as f:
        pickle.dump(out, f)


def run_sweep(tmp_path, **env):
    """Every key in a fresh process with ``env`` set; returns (results, stderr)."""
    in_path, out_path = str(tmp_path / "cases.pkl"), str(tmp_path / "results.pkl")
    with open(in_path, "wb") as f:
        pickle.dump({k: inputs(k) for k in KEYS}, f)
    code = ("import sys; sys.path.insert(0, %r); from tests import test_discrete_shapes_gpu as T; T.sweep_worker(%r, %r)"
            % (ROOT, in_path, out_path))
    e = dict(os.environ)
    for k in ("RECNN_B200_MATH", "RECNN_B200_OVERLAP", "RECNN_B200_FUSE_HEAD", "RECNN_B200_DEBUG", "RECNN_B200_GRAPHS"):
        e.pop(k, None)
    e.update(env)
    r = subprocess.run([sys.executable, "-c", code], env=e, capture_output=True, text=True, cwd=ROOT)
    assert r.returncode == 0, (r.stdout[-3000:], r.stderr[-3000:])
    with open(out_path, "rb") as f:
        return pickle.load(f), r.stderr


EPI_NAMES = {0: "HIDDEN", 1: "LINEAR", 2: "GATE", 3: "STORE", 4: "PARTIAL", 5: "ACCUM"}
_TC_LINE = re.compile(r"^\[tc_gemm\] BN=(\d+) A_MN=(\d) B_MN=(\d) EPI=(\d) M=(\d+) N=(\d+) K0=(\d+) K1=(\d+) .*"
                      r"grid=(\d+),(\d+),(\d+)")


def parse_launches(stderr):
    """{case key (strings): [(EPI, A_MN, B_MN, BN, M, N, K0, K1, splits)]} from a RECNN_B200_DEBUG=1 sweep."""
    per, cur = {}, None
    for line in stderr.splitlines():
        if line.startswith("[case] "):
            cur = tuple(line.split()[1:])
            per.setdefault(cur, [])
            continue
        m = _TC_LINE.match(line)
        if m:
            bn, amn, bmn, epi, M, N, K0, K1, _, _, gz = (int(x) for x in m.groups())
            per[cur].append((EPI_NAMES[epi], amn, bmn, bn, M, N, K0, K1, gz))
    return per


def skey(key):
    return tuple(str(x) for x in key)


def test_cuda_core_back_end(tmp_path):
    """RECNN_B200_MATH=simt: every contraction on the exact-fp32 CUDA-core kernel, the same bars, and not one
    tensor-core launch in the log."""
    res, err = run_sweep(tmp_path, RECNN_B200_MATH="simt", RECNN_B200_DEBUG="1", RECNN_B200_GRAPHS="0")
    per = parse_launches(err)
    assert set(per) == {skey(k) for k in KEYS}
    assert not any(per.values()), {k: v[:3] for k, v in per.items() if v}
    check_all(res, "simt")


def test_tensor_core_dispatch_from_the_launch_log(tmp_path):
    """RECNN_B200_DEBUG=1 logs every tensor-core launch.  The default back end takes the tensor cores exactly where
    the dispatch predicates allow at each row's chunk widths and hidden widths, and the results meet the bars."""
    res, err = run_sweep(tmp_path, RECNN_B200_DEBUG="1", RECNN_B200_GRAPHS="0")
    assert "[tc_gemm] FAILED" not in err
    per = parse_launches(err)
    assert set(per) == {skey(k) for k in KEYS}
    summary = {}
    for key in KEYS:
        launches = per[skey(key)]
        d = D.dims(key[1])
        H, widths = d["H"], D.chunk_widths(key[1])
        part = [x for x in launches if x[:3] == ("PARTIAL", 1, 1)]           # weight_grad: M = C rows of dW
        for x in launches:
            summary.setdefault(key[0], {}).setdefault("%s(%d%d)" % x[:3], set()).add(x[3])
        if key[0] == "pg":
            # dW2 of a chunk [w, H]: dZ pitch w, h pitch H; the dh GEMM contracts over w; the logits over H
            for w in widths:
                tc_dw2 = w % 4 == 0 and w >= 32 and H % 4 == 0
                assert any(x[4] == w and x[5] == H for x in part) == tc_dw2, (key, w, part)
                assert any(x[1:3] == (0, 1) and x[6] == w for x in launches) == (w % 4 == 0), (key, w)
            assert any(x[0] == "LINEAR" and x[6] == H for x in launches) == (H % 4 == 0), key
            assert any(x[4] == H for x in part) == (H % 4 == 0 and H >= 32), key                 # dW1 [H, S]
        if key[0] == "beta":
            for w in widths:
                assert any(x[4] == w for x in part) == (w % 4 == 0 and w >= 32), (key, w, part)
        if key[0] == "critic":
            # the target policy's logits of a chunk [n, w] contract over its hidden width Hp (pitch Hp); the projection
            # of a chunk, [n, H] = P W1a^T over lead + w columns, has padded operands and always takes the tensor cores;
            # the critic's dW have H rows and read [n, H] activations of pitch H
            Hp, lead = d["Hp"], d["S"] % 4
            for w in widths:
                assert any(x[0] == "LINEAR" and x[6] == Hp and x[5] == w for x in launches) == (Hp % 4 == 0), (key, w)
                assert any(x[:3] == ("PARTIAL", 0, 0) and x[5] == H and x[6] == lead + w for x in launches), (key, w)
            assert any(x[0] == "LINEAR" and x[6] == Hp for x in launches) == (Hp % 4 == 0), key
            assert any(x[4] == H for x in part) == (H % 4 == 0 and H >= 32), key
        if H % 4:
            # nothing reads a pitch-H operand on the tensor cores: no GEMM contracts over H, no dW has H rows or columns
            # (a sound test only while no other contraction length equals H: the host test keeps the table so)
            assert not any(x[0] != "PARTIAL" and x[6] == H for x in launches), (key, launches)
            assert not any(H in (x[4], x[5]) for x in part), (key, part)
        if d["n"] <= 2:
            assert all(x[8] == 1 for x in part), key
    for row in ROWS:
        if D.dims(row)["n"] >= 1000:
            for section in ("pg", "critic", "beta"):
                assert any(x[8] > 1 for k in KEYS if k[1] == row and k[0] == section for x in per[skey(k)]
                           if x[:3] == ("PARTIAL", 1, 1)), (row, section)
    bns = {x[3] for v in per.values() for x in v}
    assert bns == {64, 128}, bns
    for section, kinds in sorted(summary.items()):
        print("tensor-core launches, %s: %s" % (section, {k: sorted(v) for k, v in sorted(kinds.items())}))
    splits = sorted({x[8] for v in per.values() for x in v if x[:3] == ("PARTIAL", 1, 1)})
    print("weight_grad split counts seen: %s" % splits)
    check_all(res, "default (launch log on)")
