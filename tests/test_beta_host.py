"""Host-side checks of the Top-K notebook's behaviour policy (nn.Beta): the float64 oracle reproduces the fixtures the
unmodified notebook class produced, its closed-form backward matches float64 autograd, its RAdam step matches
torch.optim.RAdam(decoupled_weight_decay=True), the workspace stays flat in num_items once the items are chunked, and
malformed batches are refused before any device work."""
from __future__ import annotations

import ctypes

import numpy as np
import pytest
import torch

import recnn_b200
from recnn_b200 import _lib
from recnn_b200.nn.update.reinforce import _chunk_items
from oracle import beta_oracle as B
from oracle import make_beta_golden as G
from tests._golden import assert_tight_parity, load_golden


def oracle_run(name):
    """The oracle over a fixture's 7 calls: (probs, losses, sampled grads, snapshots) shaped like the fixture."""
    g = load_golden("beta_%s.npz" % name)
    inp = G.make_inputs(name)
    np.testing.assert_allclose(G.input_checksum(inp), g["input_checksum"], rtol=1e-12)
    assert np.array_equal(inp["ids"], g["ids"])
    rows = g["rows"]
    params = {"w": inp["w"].copy(), "b": inp["b"].copy()}
    o = B.make_radam()
    out = {"probs": [], "loss": [], "grad_w": [], "grad_b": [], "after_w": [], "after_b": []}
    for t in range(G.CALLS):
        p, loss, grads = B.beta_call(params, o, inp["states"][t], inp["ids"][t])
        out["probs"].append(p)
        out["loss"].append(loss)
        out["grad_w"].append(grads["w"][rows])
        out["grad_b"].append(grads["b"])
        if t + 1 in G.SNAP_AFTER:
            out["after_w"].append(params["w"][rows].copy())
            out["after_b"].append(params["b"].copy())
    return {k: np.asarray(v) for k, v in out.items()}, g, inp


def parity_dicts(got, g, inp):
    """(got, want, init) in assert_tight_parity's layout: the losses and every snapshot as a 'final' tensor."""
    want_d = {"loss.beta": g["loss"]}
    got_d = {"loss.beta": np.asarray(got["loss"], np.float64)}
    init = {}
    for i, t in enumerate(g["snap_after"]):
        name = "after%d" % t
        init[name] = {"w": inp["w"][g["rows"]], "b": inp["b"]}
        for k in ("w", "b"):
            want_d["final.%s.%s" % (name, k)] = g["after_" + k][i]
            got_d["final.%s.%s" % (name, k)] = got["after_" + k][i]
    return got_d, want_d, init


def check_against_fixture(got, g, inp, outliers=0, outlier_abs=0.0):
    """The golden bar: probabilities and losses to 1e-5, gradients within 1e-4 of the largest entry, the parameters
    after calls 1, 2, 6 and 7 through assert_tight_parity.  Returns the worst errors."""
    rep = {}
    rep["probs"] = float(np.max(np.abs(got["probs"] - g["probs"]) / (np.abs(g["probs"]) + 1e-2 * np.abs(g["probs"]).max())))
    assert rep["probs"] <= 1e-5, rep
    for k in ("grad_w", "grad_b"):
        for t in range(G.CALLS):
            scale = np.abs(g[k][t]).max()
            e = float(np.abs(got[k][t].astype(np.float64) - g[k][t]).max() / scale)
            rep[k] = max(rep.get(k, 0.0), e)
            assert e <= 1e-4, (k, t, e)
    got_d, want_d, init = parity_dicts(got, g, inp)
    rep.update(assert_tight_parity(got_d, want_d, init, outliers=outliers, outlier_abs=outlier_abs))
    return rep


@pytest.mark.parametrize("name", ["small", "ragged"])
def test_oracle_reproduces_the_notebook_fixtures(name):
    got, g, inp = oracle_run(name)
    rep = check_against_fixture(got, g, inp)
    print(name, rep)
    assert rep["checked"] == 2 * len(G.SNAP_AFTER)


def test_closed_form_matches_float64_autograd():
    rng = np.random.default_rng(3)
    n, items, S = 5, 9, 7
    w, b = rng.normal(0, 0.5, (items, S)), rng.normal(0, 0.5, items)
    s, ids = rng.normal(0, 1, (n, S)), rng.integers(0, items, n)
    p, loss, dw, db = B.loss_and_grads(w, b, s, ids)
    W = torch.tensor(w, requires_grad=True)
    bb = torch.tensor(b, requires_grad=True)
    pt = torch.softmax(torch.tensor(s) @ W.T + bb, dim=1)
    lt = torch.nn.functional.cross_entropy(pt, torch.tensor(ids))       # on the probabilities, as the notebook
    lt.backward()
    np.testing.assert_allclose(p, pt.detach().numpy(), rtol=0, atol=1e-15)
    assert abs(loss - float(lt.detach())) <= 1e-14
    np.testing.assert_allclose(dw, W.grad.numpy(), rtol=0, atol=1e-16)
    np.testing.assert_allclose(db, bb.grad.numpy(), rtol=0, atol=1e-16)


def test_expm1_form_keeps_the_signal_at_a_million_items():
    """p ~ 1/num_items: the loss and gradient from the expm1 form match float64 where the summed e^p would not."""
    items = 1 << 20
    rng = np.random.default_rng(4)
    z = rng.normal(0, 0.5, items)
    p = np.exp(z - z.max())
    p /= p.sum()
    a = 17
    p32 = p.astype(np.float32)
    em = np.expm1(p32)
    pe = np.float32(np.sum((p32 * em).astype(np.float32), dtype=np.float32))
    T = np.float32(items) + np.float32(np.sum(em, dtype=np.float32))
    g_expm1 = (em - pe) / T
    naive = np.exp(p32)
    g_naive = (naive - np.float32(np.sum(p32 * naive, dtype=np.float32))) / np.float32(np.sum(naive, dtype=np.float32))
    want = (np.exp(p) - np.sum(p * np.exp(p))) / np.sum(np.exp(p))
    scale = np.abs(want).max()
    assert np.abs(g_expm1 - want).max() <= 1e-3 * scale
    assert np.abs(g_naive - want).max() > 1e-2 * scale          # the trap the expm1 form avoids
    assert abs(float(np.log(T) - p32[a]) - float(np.log(np.sum(np.exp(p))) - p[a])) < 1e-6


@pytest.mark.parametrize("weight_decay", [0.0, 1e-2])
def test_radam_restatement_matches_torch_radam(weight_decay):
    """8 steps (un-rectified 1-5, rectified 6-8) against torch.optim.RAdam(decoupled_weight_decay=True)."""
    rng = np.random.default_rng(5)
    w0, b0 = rng.normal(0, 1, (6, 10)).astype(np.float32), rng.normal(0, 1, 6).astype(np.float32)
    params = {"w": w0.copy(), "b": b0.copy()}
    o = B.make_radam(lr=1e-2, weight_decay=weight_decay)
    tw, tb = torch.tensor(w0, requires_grad=True), torch.tensor(b0, requires_grad=True)
    opt = torch.optim.RAdam([tw, tb], lr=1e-2, weight_decay=weight_decay, decoupled_weight_decay=True)
    for _ in range(8):
        gw, gb = rng.normal(0, 1, (6, 10)).astype(np.float32), rng.normal(0, 1, 6).astype(np.float32)
        B.radam_step(o, params, {"w": gw, "b": gb})
        tw.grad, tb.grad = torch.tensor(gw), torch.tensor(gb)
        opt.step()
        for mine, theirs in ((params["w"], tw), (params["b"], tb)):
            np.testing.assert_allclose(mine, theirs.detach().numpy(), rtol=1e-6, atol=1e-7)
    assert np.abs(params["w"] - w0).max() > 1e-2                  # it did move


def test_workspace_does_not_grow_with_num_items():
    L = _lib.lib()
    sizes = []
    for items in (1 << 18, 1 << 19, 1 << 20):
        chunk = _chunk_items(2048, items)
        assert chunk == 131072
        sizes.append(L.recnn_beta_workspace_bytes(_lib.BetaDims(1290, items, (0, 0)), 2048, chunk))
    assert sizes[0] > 0 and len(set(sizes)) == 1
    # one [rows, chunk] dZ chunk and one chunk's dW partials are the large pieces; nothing is [rows, num_items]
    assert sizes[0] <= 2048 * 131072 * 4 + 131072 * 1291 * 4 + 2048 * 1292 * 4 + (1 << 20)
    d = _lib.BetaDims(1290, 5000, (0, 0))
    assert L.recnn_beta_workspace_bytes(d, 64, 100) == 0          # not a multiple of 128
    assert L.recnn_beta_workspace_bytes(d, 64, 5120) == 0         # wider than num_items
    assert L.recnn_beta_workspace_bytes(d, 64, 5000) > 0


def test_abi_mirrors_and_layout():
    L = _lib.lib()
    assert L.recnn_sizeof_beta_args() == ctypes.sizeof(_lib.BetaArgs)
    for i, f in enumerate(_lib._BETA_PROBE_FIELDS):
        assert L.recnn_offsetof_beta_args(i) == getattr(_lib.BetaArgs, f).offset, f
    buf = (ctypes.c_int64 * 4)()
    _lib.check(L.recnn_beta_layout(_lib.BetaDims(1290, 1003, (0, 0)), buf))
    assert list(buf) == [0, 1003 * 1292, 1292, 1003 * 1292 + 1004]
    assert _lib.OPT_RADAM == 4


def test_module_matches_the_notebook_class():
    beta = recnn_b200.nn.Beta(1290, 37)
    assert [k for k in beta.state_dict()] == ["net.0.weight", "net.0.bias"]
    assert isinstance(beta.net[1], torch.nn.Softmax) and isinstance(beta.criterion, torch.nn.CrossEntropyLoss)
    assert isinstance(beta.optim, recnn_b200.optim.RAdam)
    g = beta.optim.param_groups[0]
    assert (g["lr"], g["weight_decay"], g["betas"], g["eps"]) == (1e-5, 1e-5, (0.9, 0.999), 1e-8)
    eager = torch.nn.Sequential(torch.nn.Linear(1290, 37), torch.nn.Softmax(dim=1))
    beta.load_state_dict({"net." + k: v for k, v in eager.state_dict().items()})
    assert torch.equal(beta.net[0].weight, eager[0].weight)


def test_malformed_batches_are_refused_before_device_work():
    beta = recnn_b200.nn.Beta(12, 7)                 # on the CPU: any device work would raise RecnnError instead
    s = torch.zeros(4, 12)
    with pytest.raises(ValueError):
        beta(torch.zeros(4, 11), torch.tensor([0, 1, 2, 3]))            # state width
    with pytest.raises(ValueError):
        beta(torch.zeros(12), torch.tensor([0]))                       # state not 2-D
    with pytest.raises(ValueError):
        beta(s, torch.zeros(4, 6))                                     # one-hot width
    with pytest.raises(ValueError):
        beta(s, torch.zeros(3, 7))                                     # one-hot rows
    with pytest.raises(ValueError):
        beta(s, torch.tensor([0, 1, 2]))                               # id count
    with pytest.raises(ValueError):
        beta(s, torch.zeros(4))                                        # float [N]: neither one-hot nor ids
    with pytest.raises(ValueError):
        beta(s, torch.zeros(4, 7, dtype=torch.int64))                  # integer matrix
    with pytest.raises(_lib.RecnnError):
        beta(s, torch.tensor([0, 1, 2, 3]))                            # well-formed, but there is no CPU path
