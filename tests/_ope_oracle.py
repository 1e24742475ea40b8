"""float64 restatement of off-policy estimation: the exact log-softmax of a logged item under the REINFORCE policy
(DiscreteActor.log_prob) and under the behaviour policy (Beta.log_prob), from their fp32 weights, and the importance-
weighted estimators of recnn_b200.utils.metrics.off_policy_estimates, in numpy."""
from __future__ import annotations

import numpy as np


def _log_softmax_at(z, a):
    M = z.max(1)
    return z[np.arange(len(z)), a] - M - np.log(np.exp(z - M[:, None]).sum(1))


def policy_logits(w1, b1, w2, b2, state):
    """[N, num_items] logits of the DiscreteActor relu(s W1^T + b1) W2^T + b2, in float64."""
    x = np.asarray(state, dtype=np.float64)
    h = np.maximum(x @ np.asarray(w1, np.float64).T + np.asarray(b1, np.float64), 0.0)
    return h @ np.asarray(w2, np.float64).T + np.asarray(b2, np.float64)


def policy_log_prob(w1, b1, w2, b2, state, action):
    """float64 [N]: log pi(action | state)."""
    return _log_softmax_at(policy_logits(w1, b1, w2, b2, state), np.asarray(action))


def beta_log_prob(w, b, state, action):
    """float64 [N]: log beta(action | state) of Beta's Linear (w [num_items, S], b [num_items])."""
    z = np.asarray(state, np.float64) @ np.asarray(w, np.float64).T + np.asarray(b, np.float64)
    return _log_softmax_at(z, np.asarray(action))


def weights(lp_pi, lp_beta, K=1):
    """alpha_K / beta with alpha_K = 1 - (1 - pi)^K (exact in float64 for the pi the tests use)."""
    pi = np.exp(np.asarray(lp_pi, np.float64))
    alpha = pi if K == 1 else -np.expm1(K * np.log1p(-pi))
    return alpha / np.exp(np.asarray(lp_beta, np.float64))


def estimates(lp_pi, lp_beta, reward, K=1, clip=None):
    w = weights(lp_pi, lp_beta, K)
    r = np.asarray(reward, np.float64)
    n = len(r)
    wr = w * r
    out = {"ips": wr.mean(), "snips": wr.sum() / w.sum(), "ess": w.sum() ** 2 / (w * w).sum(),
           "ips_stderr": wr.std(ddof=1) / np.sqrt(n), "max_weight": w.max(), "logged_reward": r.mean(), "n": n}
    if clip is not None:
        out["clipped_ips"] = (np.minimum(w, clip) * r).mean()
        out["clipped_share"] = (w > clip).mean()
    return out
