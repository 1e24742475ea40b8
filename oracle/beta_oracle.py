"""Float64 restatement of the Top-K notebook's behaviour policy (class Beta, cell 3 of examples/2. REINFORCE TopK Off
Policy Correction/3. TopK Reinforce Off Policy Correction.ipynb): one call = forward, CrossEntropyLoss applied to the
softmax probabilities, the closed-form backward and one RAdam step.

The backward is the closed form the CUDA step uses (recnn_b200/csrc/beta.cuh), in float64:
    dL/dz_nj = (p_nj / N) ((e^{p_nj} - U_n) / T_n + p_{n,a_n} - [j == a_n]),  T = sum e^p,  U = sum p e^p.
The RAdam step is the RAdam half of the Ranger restatement (recnn_oracle._ranger_step) with Lookahead never due.
"""
from __future__ import annotations

import numpy as np

from oracle import recnn_oracle as O

F32 = np.float32
_NEVER = 1 << 62          # a Lookahead period no run reaches: Ranger's update without its slow weights


def probs(w, b, state):
    """softmax(state W^T + b) along the items, float64."""
    z = np.asarray(state, np.float64) @ np.asarray(w, np.float64).T + np.asarray(b, np.float64)
    z -= z.max(axis=1, keepdims=True)
    e = np.exp(z)
    return e / e.sum(axis=1, keepdims=True)


def loss_and_grads(w, b, state, ids):
    """(p [N, I], mean loss, dW [I, S], db [I]) of CrossEntropyLoss(p, ids), float64, via the expm1 form."""
    s = np.asarray(state, np.float64)
    p = probs(w, b, s)
    n, items = p.shape
    rows = np.arange(n)
    ids = np.asarray(ids, np.int64)
    em = np.expm1(p)
    T = items + em.sum(axis=1)
    pe = (p * em).sum(axis=1)                     # U - 1, with sum p = 1
    pa = p[rows, ids]
    loss = float(np.mean(np.log(T) - pa))
    dz = p / n * ((em - pe[:, None]) / T[:, None] + pa[:, None])
    dz[rows, ids] -= p[rows, ids] / n
    return p, loss, dz.T @ s, dz.sum(axis=0)


def make_radam(lr=1e-5, weight_decay=1e-5, betas=(0.9, 0.999), eps=1e-8):
    """torch_optimizer.RAdam's hyper-parameters (N_sma >= 5 switch: at beta2 = 0.999, N_sma > 5 is the same set of
    steps) as a Ranger restatement whose Lookahead is never due."""
    return O.make_optimizer("ranger", lr=lr, k=_NEVER, N_sma_threshhold=5, betas=betas, eps=eps,
                            weight_decay=weight_decay)


def radam_step(o, params, grads):
    """One RAdam step of params {"w", "b"} (fp32, replaced) with grads {"w", "b"}."""
    o["t"] += 1
    empty = np.zeros(0, F32)
    p = {k: empty for k in O.PARAM_ORDER}
    g = {k: empty for k in O.PARAM_ORDER}
    p["w1"], p["b1"] = params["w"], params["b"]
    g["w1"], g["b1"] = np.asarray(grads["w"], F32), np.asarray(grads["b"], F32)
    O._ranger_step(o, p, g, o["t"])
    params["w"], params["b"] = p["w1"], p["b1"]


def beta_call(params, o, state, ids):
    """One Beta.forward(state, action): returns (pre-step probs, loss, {"w": dW, "b": db}) and steps params."""
    p, loss, dw, db = loss_and_grads(params["w"], params["b"], state, ids)
    grads = {"w": dw, "b": db}
    radam_step(o, params, grads)
    return p, loss, grads
