"""Seeded synthetic cases shared by the golden generator, the tests and bench.

TEST INFRASTRUCTURE (see oracle/recnn_oracle.py header).  Every case is a pure
function of its spec; the golden fixtures store float64 checksums of the inputs
so a drift in numpy's generator would be detected rather than silently
compared against stale outputs.
"""
from __future__ import annotations

import numpy as np

from . import recnn_oracle as O

F32 = np.float32

# name -> spec.  "canon" = the reference's documented shapes (SURVEY.md 8):
# D=128, F=10, S=1290, A=128, H=256, init_w as in .circleci/tests/learning.py:20-21.
# Seeds are chosen by oracle/find_seeds.py so that, over all 12 steps and both optimizers, no kept
# hidden unit has a pre-activation closer to 0 than GATE_GUARD: the ReLU gate decisions (where the
# gradient is discontinuous) are then unambiguous at fp32 accuracy and a 1e-5 comparison is meaningful.
GATE_GUARD = 2e-6
CASES = {
    "canon": dict(seeds={"ddpg": 9, "td3": 75}, n_items=1000, dim=128, frame=10, hidden=256, n_rows=32,
                  steps=12, actor_init_w=6e-1, critic_init_w=54e-2),
    "tiny": dict(seeds={"ddpg": 1, "td3": 3}, n_items=50, dim=16, frame=4, hidden=32, n_rows=24,
                 steps=12, actor_init_w=6e-1, critic_init_w=54e-2),
}

# BASELINE.json configs[1] / configs[2] at full size (4096 rows, 26,744 items): too many ReLU gates for a
# screened seed (a handful of pre-activations per step land within rounding error of 0), so this spec is
# not a golden case; tests/test_gpu_parity.py compares it against the live oracle with a flip-tolerant bar.
FULL_SPEC = dict(seeds={"ddpg": 11, "td3": 12}, n_items=26744, dim=128, frame=10, hidden=256, n_rows=4096,
                 steps=3, actor_init_w=6e-1, critic_init_w=54e-2)


def _unscreened(seed, **kw):
    base = dict(CASES["tiny"], steps=12)
    base["seeds"] = {"ddpg": seed, "td3": seed + 1}
    base.update(kw)
    return base


# Differential cases on seeds that were NOT screened by find_seeds.py (a case with an ambiguous gate is skipped by
# its test): the reference's results are stored as tests/golden/unscreened_<id>_<algo>_<opt>.npz.
UNSCREENED = {"tiny-a": _unscreened(1001),
              "narrow": _unscreened(1002, n_rows=17, dim=8, frame=3, hidden=16, n_items=40),
              "wide": _unscreened(1003, n_rows=40, hidden=64)}

DDPG_PARAMS = dict(gamma=0.99, min_value=-10, max_value=10, policy_step=10, soft_tau=0.001)  # algo.py:103-109
TD3_PARAMS = dict(gamma=0.99, noise_std=0.5, noise_clip=3, soft_tau=0.001, policy_update=10)  # algo.py:164-174


def dims(spec):
    s = spec["dim"] * spec["frame"] + spec["frame"]
    return s, spec["dim"], spec["hidden"]          # state_dim, action_dim, hidden


def make_inputs(spec, algo="ddpg"):
    """table, items, ratings, sizes, nets, masks per step (, noise per step)."""
    rng = np.random.default_rng(spec["seeds"][algo] + (0 if algo == "ddpg" else 100003))
    s_dim, a_dim, h = dims(spec)
    table, items, ratings, _ = O.synth_frames(rng, spec["n_rows"], spec["n_items"],
                                              spec["dim"], spec["frame"])
    # two pseudo-users so `done` has an interior 1 as well
    n = spec["n_rows"]
    sizes = np.asarray([n // 3 + spec["frame"], n - n // 3 + spec["frame"]], dtype=np.int64)
    nets = {}
    pol = O.make_actor(rng, s_dim, a_dim, h, spec["actor_init_w"])
    nets["policy_net"] = pol
    nets["target_policy_net"] = O.copy_net(pol)
    if algo == "ddpg":
        val = O.make_critic(rng, s_dim, a_dim, h, spec["critic_init_w"])
        nets["value_net"] = val
        nets["target_value_net"] = O.copy_net(val)
        n_masks = 6
    else:
        for i in (1, 2):
            val = O.make_critic(rng, s_dim, a_dim, h, spec["critic_init_w"])
            nets["value_net%d" % i] = val
            nets["target_value_net%d" % i] = O.copy_net(val)
        n_masks = 8
    masks = [O.synth_masks(rng, n_masks, n, h) for _ in range(spec["steps"])]
    out = dict(table=table, items=items, ratings=ratings, sizes=sizes, nets=nets, masks=masks)
    if algo == "td3":
        out["noise"] = [(rng.standard_normal((n, a_dim)) * TD3_PARAMS["noise_std"]).astype(F32)
                        for _ in range(spec["steps"])]
    return out


def input_checksums(inp) -> np.ndarray:
    """float64 fingerprints of the regenerated inputs."""
    vals = [inp["table"].sum(dtype=np.float64), float(inp["items"].sum()),
            inp["ratings"].sum(dtype=np.float64)]
    for name in sorted(inp["nets"]):
        for k in O.PARAM_ORDER:
            vals.append(inp["nets"][name][k].sum(dtype=np.float64))
    vals.append(float(sum(int(m.sum()) for step in inp["masks"] for m in step)))
    if "noise" in inp:
        vals.append(sum(x.sum(dtype=np.float64) for x in inp["noise"]))
    return np.asarray(vals, dtype=np.float64)


def sample_index(numel: int, k: int = 512) -> np.ndarray:
    """Fixed sample positions inside a flat tensor (deterministic, seedless)."""
    if numel <= k:
        return np.arange(numel, dtype=np.int64)
    return (np.arange(k, dtype=np.int64) * 2654435761 % numel).astype(np.int64)


def net_digest(net: dict) -> dict:
    """Per-tensor: sampled values + float64 sum / abs-sum."""
    out = {}
    for k in O.PARAM_ORDER:
        flat = np.asarray(net[k], dtype=F32).reshape(-1)
        out[k + ".sample"] = flat[sample_index(flat.size)].copy()
        out[k + ".sum"] = np.float64(flat.sum(dtype=np.float64))
        out[k + ".abs"] = np.float64(np.abs(flat).sum(dtype=np.float64))
    return out
