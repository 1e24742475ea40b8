"""Host half of tests/test_discrete_shapes_gpu.py: the float64 oracles that file compares against, pinned at its edges
(K = 1, K = 2, pi(a) clamped to [eps, 1 - eps], every critic row on one item id) against torch float64 autograd of the
reference's formulas, and the shape table checked against what its docstring claims.  No kernel is launched."""
from __future__ import annotations

import numpy as np
import pytest
import torch

from oracle import cases as C
from oracle import recnn_oracle as O
from oracle import reinforce_oracle as RO
from recnn_b200 import _lib
from tests import _discrete_shapes as D

F64 = torch.float64


def _torch_policy_loss(p, state, action, blp, ret, method, K):
    """reinforce.py:16-44 with models.py:150 / :168 (corr and lambda_K carry gradient) and Categorical.log_prob (the
    probability of the action normalised and clamped to [eps, 1 - eps] of float32, the reference's dtype), restated in
    float64 autograd.  Returns (loss, parameter leaves, pi(a) leaf and its per-row loss terms)."""
    t = {k: torch.tensor(v, dtype=F64, requires_grad=True) for k, v in p.items()}
    h = torch.relu(torch.tensor(state, dtype=F64) @ t["w1"].T + t["b1"])
    probs = torch.softmax(h @ t["w2"].T + t["b2"], 1)
    pa = (probs / probs.sum(1, keepdim=True))[torch.arange(len(action)), torch.as_tensor(action)]
    R = torch.tensor(ret, dtype=F64)
    lp = torch.log(torch.clamp(pa, RO.EPS, 1.0 - RO.EPS))
    if method == RO.BASIC:
        rows = -lp * R
    else:
        corr = torch.exp(lp) / torch.exp(torch.tensor(blp, dtype=F64))
        rows = corr * -lp * R
        if method == RO.TOPK:
            rows = K * (1 - torch.exp(lp)) ** (K - 1) * rows
    return rows.sum(), t, pa, rows


def _policy_case(seed, scale):
    S, H, I, n = 7, 5, 11, 40
    rng = np.random.default_rng(seed)
    p = RO.make_discrete_actor(rng, S, I, H)
    p["w2"] = (p["w2"] * scale).astype(np.float32)
    state = rng.normal(0, 1, (n, S)).astype(np.float32)
    action = rng.integers(0, I, n)
    if scale > 1:
        probs, _ = RO.discrete_forward(p, state)
        action[::2] = probs[::2].argmax(1)
        action[1::4] = probs[1::4].argmin(1)
    blp = np.log(rng.uniform(0.01, 0.2, n)).astype(np.float32)
    ret = rng.normal(0, 1, n).astype(np.float32)
    return p, state, action, blp, ret


@pytest.mark.parametrize("scale", [1.0, 300.0], ids=["plain", "clamped"])
@pytest.mark.parametrize("method,K", [(RO.BASIC, 1), (RO.CORRECTED, 1), (RO.TOPK, 1), (RO.TOPK, 2), (RO.TOPK, 10)])
def test_policy_oracle_against_autograd(method, K, scale):
    """row_terms' closed-form dL / d log pi(a) (0 outside the clamp, dlam = 0 at K = 1, q^0 at K = 2) and
    reinforce_policy_grad's loss and gradients equal float64 autograd of the restated reference."""
    p, state, action, blp, ret = _policy_case(3 + K + 10 * method, scale)
    beta = None if method == RO.BASIC else blp
    loss, t, pa, rows = _torch_policy_loss(p, state, action, blp, ret, method, K)
    pa.retain_grad()
    loss.backward()
    pa_np = pa.detach().numpy()
    if scale > 1:
        assert (pa_np > 1 - RO.EPS).any() and (pa_np < RO.EPS).any() and ((pa_np > RO.EPS) & (pa_np < 1 - RO.EPS)).any()
    L, g, _ = RO.row_terms(pa_np, beta, ret, method, K)
    np.testing.assert_allclose(L, rows.detach().numpy(), rtol=1e-12, atol=1e-15)
    # dL / d log pi(a) = pi(a) dL / d pi(a): exactly 0 where the clamp is flat
    np.testing.assert_allclose(g, pa.grad.numpy() * pa_np, rtol=1e-9, atol=1e-12)
    assert np.all(g[(pa_np >= 1 - RO.EPS) | (pa_np <= RO.EPS)] == 0)
    want_loss, grads, _ = RO.reinforce_policy_grad(p, state, action, beta, ret, method, K)
    assert want_loss == pytest.approx(float(loss.detach()), rel=1e-12, abs=1e-14)
    for k in ("w1", "b1", "w2", "b2"):
        np.testing.assert_allclose(grads[k], t[k].grad.numpy(), rtol=1e-9, atol=1e-12 * np.abs(grads[k]).max(),
                                   err_msg=k)


@pytest.mark.parametrize("train", [False, True], ids=["eval", "train"])
def test_one_hot_critic_oracle_with_every_row_on_one_id(train):
    """value_update (the oracle the item-id critic is held to) with all rows on one item: one SGD step at lr 1 moves
    each weight by minus its gradient; loss and gradient equal float64 autograd of the critic loss."""
    S, H, I, n = 6, 8, 9, 12
    rng = np.random.default_rng(11 + train)
    pp = RO.make_discrete_actor(rng, S, I, 5)
    cp = O.make_critic(rng, S, I, H, 0.3)
    oh = np.zeros((n, I), np.float32)
    oh[:, 4] = 1
    batch = {"state": rng.normal(0, 1, (n, S)).astype(np.float32), "action": oh,
             "reward": (rng.integers(1, 6, n) - 3).astype(np.float32),
             "next_state": rng.normal(0, 1, (n, S)).astype(np.float32), "done": (rng.random(n) < 0.3).astype(np.float32)}
    masks = [(rng.random((n, H)) >= 0.5).astype(np.uint8) for _ in range(2)] if train else None
    params = dict(gamma=0.99, min_value=-10, max_value=10)
    nets = {"value_net": O.copy_net(cp), "target_value_net": O.copy_net(cp), "target_policy_net": pp}
    want_loss, want = D.critic_loss_f64(nets, batch, masks, params)
    O.reset_gate_margin()
    loss, _ = RO.value_update(batch, params, nets, {"value_optimizer": O.make_optimizer("sgd", lr=1.0)}, masks)
    assert O.GATE_MARGIN["min"] > 1e-4
    assert float(loss) == pytest.approx(want_loss, rel=1e-5)
    for k, g in want.items():
        step = cp[k].astype(np.float64) - nets["value_net"][k].astype(np.float64)
        np.testing.assert_allclose(step, g, rtol=1e-4, atol=1e-5 * np.abs(g).max(), err_msg=k)
    # only the selected action column of layer 1 has a gradient
    assert np.all(want["w1"][:, S:S + 4] == 0) and np.all(want["w1"][:, S + 5:] == 0) and np.any(want["w1"][:, S + 4])


LAST_CHUNK = {"one": 1, "w28": 28, "w30": 30, "w36": 36, "w107": 107, "tiny": 100, "h320": 3, "h128": 77, "peak": 44}


def test_shape_table_rows_are_legal_and_hit_their_edges():
    """Every row is a legal call of the three paths at its chunk width, has the last-chunk width its docstring names,
    and the table covers the edges it is meant to."""
    L = _lib.lib()
    assert set(LAST_CHUNK) == set(D.ROWS)
    for row in D.ROWS:
        d = D.dims(row)
        chunk = min(d["chunk"], d["I"])
        assert D.last_chunk(row) == LAST_CHUNK[row], row
        assert chunk == d["I"] or chunk % 128 == 0, row
        assert L.recnn_reinforce_scratch_floats(_lib.DiscreteDims(d["S"], d["H"], d["I"], 0), d["n"], chunk) > 0, row
        cd, pd = _lib.Dims(d["S"], d["I"], d["H"], 0), _lib.DiscreteDims(d["S"], d["Hp"], d["I"], 0)
        assert L.recnn_discrete_value_workspace_bytes(cd, pd, d["n"], chunk) > 0, row
        assert L.recnn_beta_workspace_bytes(_lib.BetaDims(d["S"], d["I"], (0, 0)), d["n"], chunk) > 0, row
    S = {v[0] for v in D.ROWS.values()}
    H = {v[1] for v in D.ROWS.values()}
    assert {s % 4 for s in S} == {0, 1, 2, 3}
    assert {3, 30, 36, 50, 100, 320} <= H and any(h % 64 == 0 for h in H)
    assert {1, 28, 30, 36, 107} <= set(LAST_CHUNK.values()) and any(v[3] < 128 for v in D.ROWS.values())
    assert {v[5] for v in D.ROWS.values()} == {1, 2, 129, 1000}
    assert any(v[2] != v[1] and v[2] % 4 for v in D.ROWS.values())
    # the launch-log test reads "a tensor-core GEMM contracts over H" as a K0 == H launch: with H % 4 != 0 no other
    # contraction length (S, a chunk width) and no row count may equal H.  Hp == H may (tiny): that Hp is not a
    # multiple of 4 either, so a tensor-core launch over it would be as wrong
    for row in D.ROWS:
        d = D.dims(row)
        if d["H"] % 4:
            assert d["H"] not in [d["S"], d["n"]] + D.chunk_widths(row), row
            assert d["Hp"] != d["H"] or d["Hp"] % 4, row


@pytest.mark.parametrize("row", list(D.ROWS))
def test_shape_table_seeds_keep_every_gate_unambiguous(row):
    """The recorded seeds: no gate the backward passes through within C.GATE_GUARD of 0 (policy layer 1; the online
    critic's layers over its three steps, eval and train), and no pi(a) that fp32 could place on the other side of
    the clamp."""
    inp = D.pg_inputs(row)
    assert D.pg_margin(inp) > C.GATE_GUARD
    classes = D.clamp_classes(inp)
    assert not (classes == 2).any()
    assert (row == D.PEAK_ROW) == bool((classes != 0).any())
    for train in (False, True):
        assert D.critic_oracle(D.critic_inputs(row, train), D.dims(row)["I"])[2] > C.GATE_GUARD, (row, train)
