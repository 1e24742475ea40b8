"""The shape table of tests/test_discrete_shapes_gpu.py and its host-side half: the seeded inputs of every case, the
float64 / one-hot oracles they are compared with, and the gate margins that make a tight comparison meaningful.

Every row pins a dispatch edge of the REINFORCE policy gradient (reinforce.cuh), the item-id critic step
(critic_ids.cuh) and the Beta step (beta.cuh), which share step.cu's contraction helpers.  The ragged last chunk is
num_items % chunk wide (a single chunk when num_items <= chunk); lead = S % 4 zero columns precede the projection's
chunk.  Hp is the hidden width of the critic's target policy (the critic's own width is H).

  one    S 52 (lead 0), H 64,  Hp 30,  257 items, chunk 128, 129 rows   last chunk 1 item (its dz, dW2 and dh GEMMs
                                                                         with C = 1); Hp % 4 != 0 and < 32 (the target
                                                                         policy's logits GEMM on the CUDA cores); the
                                                                         key sort pads 129 rows to 256
  w28    S 33 (lead 1), H 30,  Hp 64,  284 items, chunk 128, 2 rows     last chunk 28: % 4 == 0 but < 32, so Beta's dW of
                                                                         that chunk runs on the CUDA cores and the
                                                                         policy's dh on the tensor cores; H 30 (% 4 != 0,
                                                                         < 32): logits and every dW on the CUDA cores
  w30    S 34 (lead 2), H 36,  Hp 36,  1054 items, chunk 128, 1000 rows last chunk 30 (% 4 != 0: every GEMM that
                                                                         contracts over or reduces into that chunk on
                                                                         the CUDA cores); H 36, the first tensor-core
                                                                         width of weight_grad; split-K > 1
  w36    S 35 (lead 3), H 100, Hp 50,  292 items, chunk 128, 129 rows   last chunk 36, the first tensor-core dW2 width;
                                                                         H % 32 != 0 on the tensor cores (unfused value
                                                                         head); Hp % 4 != 0
  w107   S 25 (lead 1), H 50,  Hp 100, 1131 items, chunk 256, 129 rows  last chunk 107 (odd, 256-wide full chunks);
                                                                         H % 4 != 0 and > 32: the logits, dW2, critic
                                                                         layer 2 and every dW of H rows on the CUDA
                                                                         cores, the dh GEMM of the 256-wide chunks on
                                                                         the tensor cores
  tiny   S 2 (lead 2),  H 3,   Hp 3,   100 items, one chunk, 1 row      the smallest net: a single row (one split, a
                                                                         key array of length 1) and one chunk narrower
                                                                         than a tile
  h320   S 43 (lead 3), H 320, Hp 64,  131 items, chunk 128, 129 rows   H > 256 (the critic's head unfused, 128-wide
                                                                         tiles); last chunk 3
  h128   S 16 (lead 0), H 128, Hp 128, 77 items, one chunk, 2 rows      H a multiple of 64 on every tensor-core path;
                                                                         one chunk of 77 (% 4 != 0)
  peak   S 52 (lead 0), H 64,  Hp 64,  300 items, chunk 128, 129 rows   last chunk 44; policy logits scaled so that some
                                                                         rows have pi(a) > 1 - eps or < eps (the clamp
                                                                         of torch.distributions turns their gradient off)

The seeds (policy gradient, critic in eval mode, critic in train mode) are screened with the oracle: no pre-activation
of a gate that the backward passes through lies within C.GATE_GUARD of 0 (pg_margin, critic_margin), so the kernel and
the oracle take every ReLU decision alike."""
from __future__ import annotations

import numpy as np

from oracle import cases as C
from oracle import recnn_oracle as O
from oracle import reinforce_oracle as RO

EPS = RO.EPS
# id -> (S, H, Hp, num_items, chunk, n_rows, (pg seed, critic eval seed, critic train seed))
ROWS = {
    "one": (52, 64, 30, 257, 128, 129, (1, 1, 1)),
    "w28": (33, 30, 64, 284, 128, 2, (1, 1, 1)),
    "w30": (34, 36, 36, 1054, 128, 1000, (1, 13, 2)),
    "w36": (35, 100, 50, 292, 128, 129, (1, 2, 1)),
    "w107": (25, 50, 100, 1131, 256, 129, (1, 3, 2)),
    "tiny": (2, 3, 3, 100, 100, 1, (1, 1, 1)),
    "h320": (43, 320, 64, 131, 128, 129, (1, 22, 1)),
    "h128": (16, 128, 128, 77, 77, 2, (1, 1, 1)),
    "peak": (52, 64, 64, 300, 128, 129, (4, 1, 1)),
}
PEAK_ROW, PEAK_SCALE = "peak", 100.0
# (method name, K): every method, and K in {1, 2, 10} for Top-K (the dlam = 0 and q^0 branches, and the default)
PG_CASES = [("basic_reinforce", 10), ("reinforce_with_correction", 10), ("reinforce_with_TopK_correction", 1),
            ("reinforce_with_TopK_correction", 2), ("reinforce_with_TopK_correction", 10)]
CRITIC_STEPS = 3
CRITIC_PARAMS = dict(gamma=0.99, min_value=-10, max_value=10)
BETA_CALLS = 2
LR = 1e-3


def dims(row):
    S, H, Hp, I, chunk, n, seeds = ROWS[row]
    return dict(S=S, H=H, Hp=Hp, I=I, chunk=chunk, n=n, seeds=seeds)


def last_chunk(row):
    """Width of the last item chunk (the whole vocabulary when it fits in one)."""
    _, _, _, I, chunk, _, _ = ROWS[row]
    return I - (I - 1) // chunk * chunk


def chunk_widths(row):
    _, _, _, I, chunk, _, _ = ROWS[row]
    return sorted({min(chunk, I), last_chunk(row)})


def edge_list(I, chunk):
    last0 = (I - 1) // chunk * chunk
    return list(dict.fromkeys([I - 1, 0, last0, min(chunk - 1, I - 1), min(chunk, I - 1)]))


def edge_ids(rng, n, I, chunk):
    """Random ids with, first, the last item (the ragged last chunk's last column), item 0, the first item of the last
    chunk, the last and first columns around the first chunk boundary; then a run of repeats of earlier rows."""
    a = rng.integers(0, I, n)
    edges = edge_list(I, chunk)[:n]
    a[:len(edges)] = edges
    k = min((n - len(edges)) // 4, len(edges))
    a[len(edges):len(edges) + k] = a[:k]
    return a


# ----------------------------------------------------------------------------- policy gradient
def pg_inputs(row, seed=None):
    """Policy parameters, states, actions, behaviour log-probs and returns of the policy-gradient case of ``row``."""
    d = dims(row)
    S, H, I, chunk, n = d["S"], d["H"], d["I"], d["chunk"], d["n"]
    rng = np.random.default_rng(1000 * (seed if seed is not None else d["seeds"][0]) + S + I)
    p = RO.make_discrete_actor(rng, S, I, H)
    if row == PEAK_ROW:
        p["w2"] = (p["w2"] * PEAK_SCALE).astype(np.float32)
    state = rng.normal(0, 1, (n, S)).astype(np.float32)
    action = edge_ids(rng, n, I, chunk)
    blp = np.log(rng.uniform(1e-4, 5e-4, n)).astype(np.float32)
    ret = rng.normal(0, 1, n).astype(np.float32)
    if row == PEAK_ROW:
        # rows 8.. on their most probable item (pi(a) above 1 - eps where the logits are peaked enough) and on their
        # least probable one (below eps), alternately
        probs, _ = RO.discrete_forward(p, state)
        action[8::2] = probs[8::2].argmax(1)
        action[9::2] = probs[9::2].argmin(1)
    return {"p": p, "state": state, "action": action, "blp": blp, "ret": ret}


def pg_margin(inp):
    """Smallest |pre-activation| of the policy's hidden layer (float64): the gate of the gradient's layer-1 term."""
    z = inp["state"].astype(np.float64) @ inp["p"]["w1"].astype(np.float64).T + inp["p"]["b1"].astype(np.float64)
    return float(np.abs(z).min())


def clamp_classes(inp):
    """Per row: 0 inside (eps, 1 - eps), 1 above, -1 below, 2 too close to either end for fp32 to decide (within a
    factor 4 of 1 - pi = eps: fp32 rounds pi near 1 in steps of eps / 2; within 1e-3 relative of pi = eps)."""
    probs, _ = RO.discrete_forward(inp["p"], inp["state"])
    pa = probs[np.arange(len(inp["action"])), inp["action"]]
    out = np.zeros(len(pa), np.int64)
    out[1.0 - pa < EPS] = 1
    out[pa < EPS] = -1
    out[((1.0 - pa) > EPS / 4) & ((1.0 - pa) < 4 * EPS)] = 2
    out[np.abs(pa / EPS - 1.0) < 1e-3] = 2
    return out


def pg_oracle(inp, method, K):
    mid = RO.METHODS[method]
    loss, grads, aux = RO.reinforce_policy_grad(inp["p"], inp["state"], inp["action"],
                                                None if mid == RO.BASIC else inp["blp"], inp["ret"], mid, K)
    return loss, grads, aux


# ----------------------------------------------------------------------------- item-id critic
def critic_inputs(row, train, seed=None):
    """Target policy (hidden Hp), critic (hidden H) and, per step, a batch of item ids with its dropout masks.  Step 0
    puts every row on one id (the first item of the last chunk: the longest serial run of the action-gradient scatter),
    step 1 gives every row a distinct id (as far as the vocabulary allows) with the edge ids in front, step 2 draws only
    ids of the last, ragged chunk."""
    d = dims(row)
    S, H, Hp, I, chunk, n = d["S"], d["H"], d["Hp"], d["I"], d["chunk"], d["n"]
    rng = np.random.default_rng(1000 * (seed if seed is not None else d["seeds"][1 + int(train)]) + 7 * S + I + H)
    pp = RO.make_discrete_actor(rng, S, I, Hp)
    if row == PEAK_ROW:
        pp["w2"] = (pp["w2"] * PEAK_SCALE).astype(np.float32)
    cp = O.make_critic(rng, S, I, H, 0.3)
    last0 = (I - 1) // chunk * chunk
    batches, masks = [], []
    for step in range(CRITIC_STEPS):
        if step == 0:
            action = np.full(n, last0, np.int64)
        elif step == 1:
            edges = edge_list(I, chunk)[:n]
            rest = rng.permutation(np.setdiff1d(np.arange(I), edges))[:n - len(edges)]
            action = np.concatenate([edges, rest])
        else:
            action = rng.integers(last0, I, n)
        batches.append({"state": rng.normal(0, 1, (n, S)).astype(np.float32), "action": action.astype(np.int64),
                        "reward": (rng.integers(1, 6, n) - 3).astype(np.float32),
                        "next_state": rng.normal(0, 1, (n, S)).astype(np.float32),
                        "done": (rng.random(n) < 0.1).astype(np.float32)})
        masks.append([(rng.random((n, H)) >= 0.5).astype(np.uint8) for _ in range(2)] if train else None)
    return {"pp": pp, "cp": cp, "batches": batches, "masks": masks}


def one_hot(batch, I):
    d = dict(batch)
    oh = np.zeros((len(batch["action"]), I), np.float32)
    oh[np.arange(len(batch["action"])), batch["action"]] = 1
    d["action"] = oh
    return d


def _online_margin(v, dense, m):
    """Smallest |pre-activation| of the online critic's kept units on one batch (the gates its backward passes
    through); the target nets only run forward."""
    x = np.concatenate([dense["state"], dense["action"]], 1).astype(np.float64)
    z1 = x @ v["w1"].astype(np.float64).T + v["b1"].astype(np.float64)
    h1 = np.maximum(z1, 0) * (1.0 if m is None else 2.0 * m[0])
    z2 = h1 @ v["w2"].astype(np.float64).T + v["b2"].astype(np.float64)
    margin = float("inf")
    for z, keep in ((z1, None if m is None else m[0]), (z2, None if m is None else m[1])):
        az = np.abs(z) if keep is None else np.abs(z)[keep != 0]
        if az.size:
            margin = min(margin, float(az.min()))
    return margin


def critic_oracle(inp, I):
    """value_update on the dense one-hot for CRITIC_STEPS Adam steps: (losses, final critic, gate margin of the online
    critic over the run's steps)."""
    nets = {"value_net": O.copy_net(inp["cp"]), "target_value_net": O.copy_net(inp["cp"]),
            "target_policy_net": inp["pp"]}
    opts = {"value_optimizer": O.make_optimizer("adam", lr=LR)}
    losses, margin = [], float("inf")
    for b, m in zip(inp["batches"], inp["masks"]):
        dense = one_hot(b, I)
        margin = min(margin, _online_margin(nets["value_net"], dense, m))
        loss, _ = RO.value_update(dense, CRITIC_PARAMS, nets, opts, m, learn=True)
        losses.append(float(loss))
    return np.asarray(losses), nets["value_net"], margin


def critic_loss_f64(nets, batch, masks, params=None):
    """misc.py:28-41 with the dense one-hot action [N, num_items], float64 autograd w.r.t. the online critic: (loss,
    {w1, b1, w2, b2, w3, b3: gradient})."""
    import torch
    params = CRITIC_PARAMS if params is None else params
    f = lambda a: torch.tensor(a, dtype=torch.float64)                                # noqa: E731
    v = {k: torch.tensor(a, dtype=torch.float64, requires_grad=True) for k, a in nets["value_net"].items()}
    tv, tp = ({k: f(a) for k, a in nets[n].items()} for n in ("target_value_net", "target_policy_net"))
    s, s2, a = f(batch["state"]), f(batch["next_state"]), f(batch["action"])
    r, d = f(batch["reward"])[:, None], f(batch["done"])[:, None]
    probs = torch.softmax(torch.relu(s2 @ tp["w1"].T + tp["b1"]) @ tp["w2"].T + tp["b2"], 1)

    def critic(net, x, act, m=None):
        h = torch.relu(torch.cat([x, act], 1) @ net["w1"].T + net["b1"])
        if m is not None:
            h = h * 2 * f(m[0])
        h = torch.relu(h @ net["w2"].T + net["b2"])
        if m is not None:
            h = h * 2 * f(m[1])
        return h @ net["w3"].T + net["b3"]

    y = (r + (1 - d) * params["gamma"] * critic(tv, s2, probs)).clamp(params["min_value"], params["max_value"])
    loss = ((critic(v, s, a, masks) - y) ** 2).mean()
    loss.backward()
    return float(loss.detach()), {k: t.grad.numpy() for k, t in v.items()}


def neutralise_gates(v, dense, m):
    """Copies of the dropout masks m with every kept unit whose pre-activation lies within C.GATE_GUARD of 0 dropped
    (layer 1 first, then layer 2 on the thinned layer 1), so that no gate of the backward is ambiguous at fp32."""
    m1, m2 = m[0].copy(), m[1].copy()
    x = np.concatenate([dense["state"], dense["action"]], 1).astype(np.float64)
    z1 = x @ v["w1"].astype(np.float64).T + v["b1"].astype(np.float64)
    m1[np.abs(z1) <= C.GATE_GUARD] = 0
    z2 = (np.maximum(z1, 0) * 2.0 * m1) @ v["w2"].astype(np.float64).T + v["b2"].astype(np.float64)
    m2[np.abs(z2) <= C.GATE_GUARD] = 0
    return [m1, m2]


def grad_batches(inp, I):
    """The batches of the gradient check at the initial weights: in train mode every batch of critic_inputs, with its
    masks neutralised (neutralise_gates); in eval mode the all-rows-on-one-id batch, whose gates the seed screening
    covers (it is the first step of critic_oracle).  [(batch, masks or None)]"""
    if inp["masks"][0] is None:
        return [(inp["batches"][0], None)]
    return [(b, neutralise_gates(inp["cp"], one_hot(b, I), m)) for b, m in zip(inp["batches"], inp["masks"])]


def critic_grads_f64(inp, I):
    """(loss, gradient) of the critic loss at the initial weights for each of grad_batches, float64 autograd."""
    nets = {"value_net": inp["cp"], "target_value_net": inp["cp"], "target_policy_net": inp["pp"]}
    return [critic_loss_f64(nets, one_hot(b, I), m) for b, m in grad_batches(inp, I)]


# ----------------------------------------------------------------------------- Beta
def beta_inputs(row):
    """Weights, and per call states and target ids (edge ids: the last item, in the one-item chunk of row "one")."""
    d = dims(row)
    S, I, chunk, n = d["S"], d["I"], d["chunk"], d["n"]
    rng = np.random.default_rng(S + I + n)
    bound = 1.0 / np.sqrt(S)
    w = rng.uniform(-bound, bound, (I, S)).astype(np.float32)
    b = rng.uniform(-bound, bound, I).astype(np.float32)
    calls = [(rng.normal(0, 1, (n, S)).astype(np.float32), edge_ids(rng, n, I, chunk)) for _ in range(BETA_CALLS)]
    return {"w": w, "b": b, "calls": calls}


def beta_oracle(inp):
    """beta_call for each call: (probs, losses, grads, final params)."""
    from oracle import beta_oracle as B
    params = {"w": inp["w"].copy(), "b": inp["b"].copy()}
    o = B.make_radam()
    probs, losses, grads = [], [], []
    for s, ids in inp["calls"]:
        p, loss, g = B.beta_call(params, o, s, ids)
        probs.append(p)
        losses.append(loss)
        grads.append(g)
    return probs, np.asarray(losses), grads, params


def screen(limit=200):
    """First seeds (per row: policy gradient, critic eval, critic train) whose margins clear C.GATE_GUARD."""
    out = {}
    for row in ROWS:
        found = []
        for kind in ("pg", "eval", "train"):
            for seed in range(1, limit):
                if kind == "pg":
                    inp = pg_inputs(row, seed)
                    ok = pg_margin(inp) > C.GATE_GUARD and not (clamp_classes(inp) == 2).any()
                else:
                    ok = critic_oracle(critic_inputs(row, kind == "train", seed), ROWS[row][3])[2] > C.GATE_GUARD
                if ok:
                    found.append(seed)
                    break
            else:
                found.append(None)
        out[row] = tuple(found)
        print(row, out[row], flush=True)
    return out


if __name__ == "__main__":
    screen()
