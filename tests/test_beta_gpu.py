"""The Top-K notebook's behaviour policy (nn.Beta -> recnn_beta_step) on the GPU: against the fixtures of the unmodified
notebook class, against the live float64 oracle at unaligned shapes with forced chunking on both GEMM back ends,
one-hot / item-id / repeat / external-optimizer equivalences, zero pitch pads, a million items with bounded memory,
the notebook's Reinforce wiring end to end, and the error paths."""
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
from recnn_b200.nn import beta as BM
from recnn_b200.nn.arena import param_arena, grad_arena
from recnn_b200.nn.update import reinforce as RF
from oracle import beta_oracle as B
from oracle import make_beta_golden as G
from tests._golden import assert_tight_parity, load_golden
from tests.test_beta_host import check_against_fixture

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
# chunked vs single chunk: only the order of the softmax sums (merged per chunk) and the split-K order of dW differ
REORDER_BAR = 1e-5


def make_beta(w, b, optim=None):
    items, S = w.shape
    beta = recnn_b200.nn.Beta(S, items)
    beta.load_state_dict({"net.0.weight": torch.from_numpy(w), "net.0.bias": torch.from_numpy(b)})
    return beta.to(DEV)


def force_chunk(monkeypatch, chunk):
    monkeypatch.setattr(BM, "_chunk_items", lambda rows, items: items if chunk is None else min(chunk, items))


def onehot(ids, items):
    a = torch.zeros(len(ids), items, device=DEV)
    a[torch.arange(len(ids)), torch.as_tensor(ids, device=DEV)] = 1.0
    return a


def snapshot(beta):
    """(probs-independent) state of a Beta after a call: parameters, .grad and the RAdam arenas, as float64 arrays."""
    lin = beta.net[0]
    out = {"w": lin.weight.detach().double().cpu().numpy(), "b": lin.bias.detach().double().cpu().numpy(),
           "gw": lin.weight.grad.double().cpu().numpy(), "gb": lin.bias.grad.double().cpu().numpy()}
    if isinstance(beta.optim, recnn_b200.optim.RAdam):
        out["m"] = beta.optim._m.cpu().numpy().copy()
        out["v"] = beta.optim._v.cpu().numpy().copy()
        out["t"] = int(beta.optim._t.item())
    return out


def native_fixture_run(name, form="onehot"):
    inp = G.make_inputs(name)
    g = load_golden("beta_%s.npz" % name)
    rows = g["rows"]
    beta = make_beta(inp["w"], inp["b"])
    items = inp["w"].shape[0]
    out = {"probs": [], "loss": [], "grad_w": [], "grad_b": [], "after_w": [], "after_b": []}
    for t in range(G.CALLS):
        ids = torch.from_numpy(inp["ids"][t]).to(DEV)
        p = beta(torch.from_numpy(inp["states"][t]).to(DEV), onehot(ids, items) if form == "onehot" else ids)
        out["probs"].append(p.cpu().numpy())
        out["loss"].append(float(beta.last_loss))
        out["grad_w"].append(beta.net[0].weight.grad[torch.from_numpy(rows)].cpu().numpy())
        out["grad_b"].append(beta.net[0].bias.grad.cpu().numpy())
        if t + 1 in G.SNAP_AFTER:
            out["after_w"].append(beta.net[0].weight.detach()[torch.from_numpy(rows)].cpu().numpy())
            out["after_b"].append(beta.net[0].bias.detach().cpu().numpy())
    return {k: np.asarray(v) for k, v in out.items()}, g, inp


@pytest.mark.parametrize("name", ["small", "ragged"])
def test_golden_fixtures(name):
    """7 calls through the public API with one-hot actions, against what the notebook's class produced."""
    got, g, inp = native_fixture_run(name)
    rep = check_against_fixture(got, g, inp)
    print(name, rep)


def edge_ids(rng, n, items, chunk):
    ids = rng.integers(0, items, n)
    edges = [0, items - 1]
    if chunk < items:
        edges += [chunk - 1, chunk, (items - 1) // chunk * chunk]
    ids[:len(edges)] = edges
    return ids


def oracle_sweep_case(S, items, n, chunk, calls=3, seed=0, form="onehot"):
    """`calls` native calls against the live float64 oracle; returns the worst errors and the final snapshot."""
    rng = np.random.default_rng(seed + S + items)
    bound = 1.0 / np.sqrt(S)
    w = rng.uniform(-bound, bound, (items, S)).astype(np.float32)
    b = rng.uniform(-bound, bound, items).astype(np.float32)
    beta = make_beta(w, b)
    params = {"w": w.copy(), "b": b.copy()}
    o = B.make_radam()
    rep = {"probs": 0.0, "loss": 0.0, "grad_w": 0.0, "grad_b": 0.0}
    probs_all = []
    for t in range(calls):
        s = rng.normal(0, 1, (n, S)).astype(np.float32)
        ids = edge_ids(rng, n, items, chunk)
        tid = torch.from_numpy(ids).to(DEV)
        p = beta(torch.from_numpy(s).to(DEV), onehot(tid, items) if form == "onehot" else tid).double().cpu().numpy()
        probs_all.append(p)
        want_p, want_l, grads = B.beta_call(params, o, s, ids)
        rep["probs"] = max(rep["probs"], float(np.max(np.abs(p - want_p) / (want_p + 1e-2 * want_p.max()))))
        rep["loss"] = max(rep["loss"], abs(float(beta.last_loss) - want_l) / (abs(want_l) + 0.1))
        snap = snapshot(beta)
        for k, gk in (("grad_w", "gw"), ("grad_b", "gb")):
            want = grads[k[-1]]
            rep[k] = max(rep[k], float(np.abs(snap[gk] - want).max() / np.abs(want).max()))
    got_d = {"final.beta.w": snap["w"].astype(np.float32), "final.beta.b": snap["b"].astype(np.float32)}
    want_d = {"final.beta.w": params["w"], "final.beta.b": params["b"]}
    rep.update(assert_tight_parity(got_d, want_d, {"beta": {"w": w, "b": b}}))
    assert rep["probs"] <= 1e-5 and rep["loss"] <= 1e-5, rep
    assert rep["grad_w"] <= 1e-4 and rep["grad_b"] <= 1e-4, rep
    return rep, snap, np.stack(probs_all)


SWEEP = [(1290, 5000, 64, 1024), (37, 1003, 33, 128), (2570, 300, 48, 128)]


def run_sweep():
    """Every SWEEP shape chunked (ragged last chunk) and in one chunk: each against the oracle, and the two against each
    other at fp32-reordering level."""
    import _pytest.monkeypatch
    mp = _pytest.monkeypatch.MonkeyPatch()
    try:
        for S, items, n, chunk in SWEEP:
            assert items % chunk != 0
            res = {}
            for c in (chunk, None):
                force_chunk(mp, c)
                rep, snap, probs = oracle_sweep_case(S, items, n, chunk)
                print("S=%d I=%d N=%d chunk=%s: %s" % (S, items, n, c, rep))
                res[c] = (snap, probs)
            (a, pa), (b, pb) = res[chunk], res[None]
            assert np.abs(pa - pb).max() <= REORDER_BAR * pb.max()
            for k in ("w", "b", "gw", "gb"):
                assert np.abs(a[k] - b[k]).max() <= REORDER_BAR * np.abs(b[k]).max(), k
    finally:
        mp.undo()


def test_shape_sweep_against_the_oracle():
    run_sweep()


def test_shape_sweep_on_the_cuda_core_back_end():
    """The same sweep with every GEMM on the exact-fp32 CUDA-core kernel, in a process of its own (the back end is fixed
    per process)."""
    code = "import sys; sys.path.insert(0, %r); from tests import test_beta_gpu as T; T.run_sweep()" % ROOT
    env = dict(os.environ, RECNN_B200_MATH="simt")
    r = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, cwd=ROOT)
    print(r.stdout[-3000:], r.stderr[-3000:])
    assert r.returncode == 0


def _seven_calls(monkeypatch, form, chunk=128, S=37, items=1003, n=40, optim=None):
    force_chunk(monkeypatch, chunk)
    rng = np.random.default_rng(11)
    w = rng.uniform(-0.1, 0.1, (items, S)).astype(np.float32)
    b = rng.uniform(-0.1, 0.1, items).astype(np.float32)
    beta = make_beta(w, b)
    if optim is not None:
        beta.optim = optim(beta)
    probs, losses = [], []
    for t in range(7):
        s = torch.from_numpy(rng.normal(0, 1, (n, S)).astype(np.float32)).to(DEV)
        ids = torch.from_numpy(edge_ids(rng, n, items, chunk)).to(DEV)
        probs.append(beta(s, onehot(ids, items) if form == "onehot" else ids).cpu().numpy())
        losses.append(float(beta.last_loss))
    return beta, np.stack(probs), losses, snapshot(beta)


def test_onehot_ids_and_repeats_are_bit_identical(monkeypatch):
    runs = [_seven_calls(monkeypatch, f) for f in ("onehot", "ids", "ids")]
    (_, p0, l0, s0) = runs[0]
    for _, p, l, s in runs[1:]:
        assert np.array_equal(p, p0) and l == l0
        for k in s0:
            assert np.array_equal(np.asarray(s[k]), np.asarray(s0[k])), k
    assert s0["t"] == 7


def test_builtin_and_external_radam_agree(monkeypatch):
    ext = lambda beta: torch.optim.RAdam(beta.net.parameters(), lr=1e-5, weight_decay=1e-5,  # noqa: E731
                                         decoupled_weight_decay=True)
    beta0, p0, l0, s0 = _seven_calls(monkeypatch, "ids")
    beta1, p1, l1, s1 = _seven_calls(monkeypatch, "ids", optim=ext)
    rng = np.random.default_rng(11)
    w = rng.uniform(-0.1, 0.1, (1003, 37)).astype(np.float32)
    b = rng.uniform(-0.1, 0.1, 1003).astype(np.float32)
    got = {"final.beta.w": s0["w"].astype(np.float32), "final.beta.b": s0["b"].astype(np.float32)}
    want = {"final.beta.w": s1["w"].astype(np.float32), "final.beta.b": s1["b"].astype(np.float32)}
    print(assert_tight_parity(got, want, {"beta": {"w": w, "b": b}}))
    np.testing.assert_allclose(l0, l1, rtol=1e-5)


def test_pitch_pads_stay_zero(monkeypatch):
    """S = 37 (row pitch 40) and 1003 items (bias segment 1004): every pad of the parameter, gradient and moment arenas
    is exactly 0 after 7 steps."""
    beta, _, _, _ = _seven_calls(monkeypatch, "ids")
    flat, g = param_arena(beta), grad_arena(beta)
    for name, arena in (("params", flat), ("grads", g), ("m", beta.optim._m), ("v", beta.optim._v)):
        a = arena.cpu()
        w = a[:1003 * 40].view(1003, 40)
        assert torch.count_nonzero(w[:, 37:]) == 0, name
        assert torch.count_nonzero(a[1003 * 40 + 1003:]) == 0, name
        assert torch.count_nonzero(w[:, :37]) > 0, name


def test_expm1_term_carries_the_gradient_when_the_target_is_improbable(monkeypatch):
    """Targets whose bias is -60 have p_a ~ 0, so every dL/dz is the (e^p - U) / T term, of order 1/num_items^2: at
    262,144 items it is what the expm1 form keeps and e^p - 1 in fp32 would blur (its rounding is ~2% of the term)."""
    force_chunk(monkeypatch, 65536)
    rng = np.random.default_rng(21)
    S, items, n = 37, 262144, 64
    w = rng.uniform(-0.16, 0.16, (items, S)).astype(np.float32)
    b = rng.uniform(-0.16, 0.16, items).astype(np.float32)
    ids = rng.integers(0, items, n)
    ids[:4] = [0, items - 1, 65535, 65536]
    b[ids] = -60.0
    beta = make_beta(w, b)
    s = rng.normal(0, 1, (n, S)).astype(np.float32)
    p = beta(torch.from_numpy(s).to(DEV), torch.from_numpy(ids).to(DEV))
    want_p, want_l, dw, db = B.loss_and_grads(w, b, s, ids)
    snap = snapshot(beta)
    ew = float(np.abs(snap["gw"] - dw).max() / np.abs(dw).max())
    eb = float(np.abs(snap["gb"] - db).max() / np.abs(db).max())
    print("dW %.2e db %.2e of max; loss %.8f want %.8f" % (ew, eb, float(beta.last_loss), want_l))
    assert ew <= 1e-4 and eb <= 1e-4
    assert abs(float(beta.last_loss) - want_l) <= 1e-5 * (abs(want_l) + 0.1)
    assert float((p.double().cpu() - torch.from_numpy(want_p)).abs().max()) <= 1e-5 * want_p.max()


def _float64_reference(beta, state, ids, sample_rows, item_chunk=131072, row_block=512):
    """Loss, probabilities of the first rows and dW / db of sample item rows, float64 on the GPU, without a dense
    [rows, num_items] float64 matrix of all rows (two passes over item chunks per row block)."""
    W, b = beta.net[0].weight.detach(), beta.net[0].bias.detach()
    items = W.shape[0]
    n = state.shape[0]
    rs = torch.as_tensor(sample_rows, device=DEV)
    Ws = W[rs].double()
    loss, dws, dbs, p_first = 0.0, torch.zeros_like(Ws), torch.zeros(len(sample_rows), device=DEV, dtype=torch.float64), None
    for r0 in range(0, n, row_block):
        s = state[r0:r0 + row_block].double()
        a = ids[r0:r0 + row_block]
        m = torch.full((s.shape[0],), -torch.inf, device=DEV, dtype=torch.float64)
        tot = torch.zeros_like(m)
        for c0 in range(0, items, item_chunk):
            z = s @ W[c0:c0 + item_chunk].double().T + b[c0:c0 + item_chunk].double()
            mn = torch.maximum(m, z.max(1).values)
            tot = tot * torch.exp(m - mn) + torch.exp(z - mn[:, None]).sum(1)
            m = mn
        s1, s2 = torch.zeros_like(m), torch.zeros_like(m)
        pa = torch.zeros_like(m)
        for c0 in range(0, items, item_chunk):
            z = s @ W[c0:c0 + item_chunk].double().T + b[c0:c0 + item_chunk].double()
            p = torch.exp(z - m[:, None]) / tot[:, None]
            if r0 == 0 and c0 == 0:
                p_first = p[:8, :256].clone()
            em = torch.expm1(p)
            s1 += em.sum(1)
            s2 += (p * em).sum(1)
            inside = (a >= c0) & (a < c0 + p.shape[1])
            pa[inside] = p[inside, (a[inside] - c0)]
            del z, p, em
        T = items + s1
        loss += float((torch.log(T) - pa).sum())
        ps = torch.exp(s @ Ws.T + b[rs].double() - m[:, None]) / tot[:, None]
        dz = ps / n * ((torch.expm1(ps) - s2[:, None]) / T[:, None] + pa[:, None])
        dz -= (a[:, None] == rs[None, :]).double() * ps / n
        dws += dz.T @ s
        dbs += dz.sum(0)
    return loss / n, dws, dbs, p_first


def _big_case(n, S, items, seed):
    gc.collect()                     # nets of earlier tests (module <-> optimizer cycles) hold device memory until then
    torch.cuda.empty_cache()
    g = torch.Generator(device=DEV).manual_seed(seed)
    torch.manual_seed(seed)
    with torch.device(DEV):
        beta = recnn_b200.nn.Beta(S, items)
    state = torch.randn(n, S, device=DEV, generator=g)
    ids = torch.randint(0, items, (n,), device=DEV, generator=g)
    ids[:4] = torch.tensor([0, items - 1, 131071, 131072], device=DEV) % items
    return beta, state, ids


def _check_big(beta, state, ids, chunk):
    n, items = state.shape[0], beta.net[0].out_features
    sample = sorted({0, 1, chunk - 1, chunk, items - 1, int(ids[0]), int(ids[1]), int(ids[5]), 4097})
    beta.optim = torch.optim.SGD(beta.net.parameters(), lr=0.0)     # keeps the weights: the reference sees them
    p = beta(state, ids)
    want_loss, dws, dbs, p_first = _float64_reference(beta, state, ids, sample)
    got_loss = float(beta.last_loss)
    print("loss %.8f want %.8f" % (got_loss, want_loss))
    assert abs(got_loss - want_loss) <= 1e-5 * (abs(want_loss) + 0.1)
    assert float((p[:8, :256].double() - p_first).abs().max()) <= 1e-5 * float(p_first.max())
    gw = beta.net[0].weight.grad[torch.as_tensor(sample, device=DEV)].double()
    gb = beta.net[0].bias.grad[torch.as_tensor(sample, device=DEV)].double()
    ew = float((gw - dws).abs().max() / dws.abs().max())
    eb = float((gb - dbs).abs().max() / dbs.abs().max())
    print("grad rows %s: dW %.2e db %.2e of max" % (sample, ew, eb))
    assert ew <= 1e-4 and eb <= 1e-4


def _builtin_peak(beta, state, ids):
    """One call with the built-in RAdam; returns (pre-step probs of the first rows, peak bytes above the resident nets
    and arenas)."""
    beta.optim = recnn_b200.optim.RAdam(beta.net.parameters(), lr=1e-5, weight_decay=1e-5)
    beta.optim.c_net(beta)                      # the moment arenas exist before the measurement
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    p = beta(state, ids)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    # it stepped (at a million items one lr = 1e-5 step of an un-rectified RAdam is below the weights' rounding)
    assert beta.optim.steps_taken() == 1 and torch.count_nonzero(beta.optim._m[:1 << 20]) > 0
    return p[:4].clone(), peak, int(p.numel()) * 4


def test_262144_items_with_automatic_chunking(monkeypatch):
    monkeypatch.setattr(RF, "_LOGITS_BUDGET_BYTES", 128 << 20)
    n, S, items = 512, 1290, 262144
    chunk = RF._chunk_items(n, items)
    assert chunk == 65536
    beta, state, ids = _big_case(n, S, items, 3)
    _, peak, probs_bytes = _builtin_peak(beta, state, ids)
    ws = _lib.lib().recnn_beta_workspace_bytes(beta.dims, n, chunk)
    print("262144 items: peak %.1f MB above the arenas (probs %.1f MB, workspace %.1f MB)"
          % (peak / 1e6, probs_bytes / 1e6, ws / 1e6))
    assert peak <= probs_bytes + ws + (16 << 20)
    _check_big(beta, state, ids, chunk)


def million_item_memory():
    """One built-in call at 1M items x 2048 rows from a fresh allocator: what it holds at its peak."""
    n, S, items = 2048, 1290, 1 << 20
    chunk = RF._chunk_items(n, items)
    assert chunk == 131072
    beta, state, ids = _big_case(n, S, items, 4)
    _, peak, probs_bytes = _builtin_peak(beta, state, ids)
    total = torch.cuda.max_memory_allocated()
    chunk_bytes = n * chunk * 4 + chunk * (S + 1) * 4 + n * 1292 * 4
    arenas = 4 * param_arena(beta).numel() * 4
    print("1M items x 2048 rows: peak %.2f GB above the arenas, %.2f GB in all (arenas %.2f GB, probs %.2f GB)"
          % (peak / 1e9, total / 1e9, arenas / 1e9, probs_bytes / 1e9))
    assert peak <= probs_bytes + chunk_bytes + (64 << 20)
    # everything: the weights and the three other arenas, probs_out, one chunk and the batch itself
    assert total <= arenas + probs_bytes + chunk_bytes + n * S * 4 + (256 << 20)


def test_million_items_2048_rows():
    """The memory bound in a process of its own (nothing of earlier tests in the allocator), then a call that keeps the
    weights (SGD with lr = 0) against the chunked float64 reference."""
    code = "import sys; sys.path.insert(0, %r); from tests import test_beta_gpu as T; T.million_item_memory()" % ROOT
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, cwd=ROOT)
    print(r.stdout[-2000:], r.stderr[-2000:])
    assert r.returncode == 0
    n, S, items = 2048, 1290, 1 << 20
    beta, state, ids = _big_case(n, S, items, 4)
    _check_big(beta, state, ids, RF._chunk_items(n, items))


def _notebook_agent(form, items=5000, H=2048, S=1290, N=10, steps=11):
    torch.manual_seed(9)
    rng = np.random.default_rng(9)
    beta_net = recnn_b200.nn.Beta(S, items).to(DEV)
    value_net = recnn_b200.nn.Critic(S, items, H, 54e-2).to(DEV)
    policy_net = recnn_b200.nn.DiscreteActor(S, items, H).to(DEV)
    policy_net.action_source = {"pi": "beta", "beta": "beta"}
    reinforce = recnn_b200.nn.Reinforce(policy_net, value_net).to(torch.device(DEV))
    seen = []

    def beta_forward(state, action):
        p = beta_net.forward(state, action)
        seen.append(p.clone())
        return p

    def select_action_corr(state, action, K, writer, step, **kwargs):
        out = reinforce.nets["policy_net"]._select_action_with_TopK_correction(state, beta_forward, action, K=K,
                                                                              writer=writer, step=step)
        rec = reinforce.nets["policy_net"]._saved[-1]
        lp = torch.distributions.Categorical(probs=seen[-1]).log_prob(rec["action"])
        torch.testing.assert_close(rec["beta_log_prob"], lp, rtol=1e-5, atol=1e-5)
        return out

    reinforce.nets["policy_net"].select_action = select_action_corr
    reinforce.params["reinforce"] = recnn_b200.nn.ChooseREINFORCE(
        recnn_b200.nn.ChooseREINFORCE.reinforce_with_TopK_correction)
    reinforce.params["K"] = 10
    w0 = beta_net.net[0].weight.detach().clone()
    losses = []
    for _ in range(steps):
        ids = rng.integers(0, items, N)
        action = torch.from_numpy(ids) if form == "ids" else torch.from_numpy(np.eye(items, dtype=np.float32)[ids])
        b = {"state": torch.from_numpy(rng.normal(0, 1, (N, S)).astype(np.float32)), "action": action,
             "reward": torch.from_numpy(rng.integers(1, 6, N).astype(np.float32) - 3),
             "next_state": torch.from_numpy(rng.normal(0, 1, (N, S)).astype(np.float32)),
             "done": torch.from_numpy((rng.random(N) < 0.1).astype(np.float32))}
        losses.append(reinforce.update(b))
        reinforce.step()
    assert len(seen) == steps and beta_net.optim.steps_taken() == steps
    assert float((beta_net.net[0].weight.detach() - w0).abs().max()) > 0
    assert [l is not None for l in losses] == [i == 10 for i in range(steps)]
    return losses, beta_net.net[0].weight.detach().clone()


def test_notebook_wiring_end_to_end():
    l1, w1 = _notebook_agent("onehot")
    l2, w2 = _notebook_agent("ids")
    assert torch.equal(w1, w2)                 # one-hot and item-id batches drive beta identically
    print("policy step losses:", l1[-1], l2[-1])


def test_error_paths(monkeypatch):
    force_chunk(monkeypatch, 128)
    rng = np.random.default_rng(2)
    items, S, n = 1003, 37, 16
    beta = make_beta(rng.uniform(-0.1, 0.1, (items, S)).astype(np.float32), rng.uniform(-0.1, 0.1, items).astype(np.float32))
    s = torch.from_numpy(rng.normal(0, 1, (n, S)).astype(np.float32)).to(DEV)
    ids = torch.from_numpy(rng.integers(0, items, n)).to(DEV)
    beta(s, ids)
    before = snapshot(beta)
    flat0 = param_arena(beta).clone()
    for bad in (items, -1):
        ids2 = ids.clone()
        ids2[5] = bad
        with pytest.raises(IndexError):
            beta(s, ids2)
        after = snapshot(beta)
        assert torch.equal(param_arena(beta), flat0)
        for k in ("m", "v", "t"):
            assert np.array_equal(np.asarray(after[k]), np.asarray(before[k])), k
    with pytest.raises(ValueError):
        beta(s, torch.zeros(n, items - 1, device=DEV))
    with pytest.raises(ValueError):
        beta(s, ids[:-1])
    cpu = recnn_b200.nn.Beta(S, items)
    with pytest.raises(_lib.RecnnError):
        cpu(s.cpu(), ids.cpu())
    beta(s, ids)                              # still usable after the refused calls
    assert beta.optim.steps_taken() == 2


def test_dropping_a_beta_frees_its_device_memory():
    """A Beta does not sit in a reference cycle with its optimizer: its arenas and workspace leave the device as soon as
    the last reference goes, without the garbage collector."""
    gc.collect()
    start = torch.cuda.memory_allocated()
    gc.disable()
    try:
        rng = np.random.default_rng(1)
        beta = make_beta(rng.uniform(-0.1, 0.1, (3000, 64)).astype(np.float32), np.zeros(3000, np.float32))
        beta(torch.randn(32, 64, device=DEV), torch.randint(0, 3000, (32,), device=DEV))
        assert beta.optim.steps_taken() == 1
        assert torch.cuda.memory_allocated() > start + 4 * 3000 * 64 * 4
        del beta
        assert torch.cuda.memory_allocated() == start
    finally:
        gc.enable()
