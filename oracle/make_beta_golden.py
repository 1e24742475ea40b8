"""Generate tests/golden/beta_{small,ragged}.npz by running the UNMODIFIED class Beta of the reference's Top-K notebook.

Run in the build container only (needs /root/reference):

    python -m oracle.make_beta_golden

The notebook (examples/2. REINFORCE TopK Off Policy Correction/3. TopK Reinforce Off Policy Correction.ipynb) is read
as JSON and its cell 3 -- ``class Beta`` -- is exec'd as it stands, with ``nn`` = torch.nn, a small ``num_items`` and
``optim`` bound to a stand-in module whose ``RAdam`` builds ``torch.optim.RAdam(decoupled_weight_decay=True)``
(torch_optimizer is not installed; oracle/ref_import.py stubs it as an empty module).  Nothing of the notebook is
stored: only the inputs' recipe and what the calls produced.

The cell fixes S = 1290.  Each case starts from parameters drawn from a seeded numpy generator (loaded through
``load_state_dict``) and makes 7 calls on seeded states and one-hot actions, so that RAdam runs both its un-rectified
(steps 1-5) and its rectified branch (6, 7).  Stored: the targets, the pre-step probabilities and the loss of every
call (the loss by a forward hook on ``criterion``), ``.grad`` after every call and the parameters after calls 1, 2, 6 and 7 --
weights on a fixed sample of item rows (full tensors would not be small test vectors), biases whole.
"""
from __future__ import annotations

import json
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle.ref_import import REFERENCE_ROOT  # noqa: E402

GOLDEN_DIR = os.path.join(ROOT, "tests", "golden")
NOTEBOOK = os.path.join("examples", "2. REINFORCE TopK Off Policy Correction",
                        "3. TopK Reinforce Off Policy Correction.ipynb")
S = 1290
CALLS = 7
SNAP_AFTER = (1, 2, 6, 7)
CASES = {
    # name: (num_items, rows per call, sampled weight rows)
    "small": (37, 16, (0, 5, 11, 17, 23, 29, 35, 36)),
    "ragged": (300, 24, (0, 127, 128, 255, 256, 299)),
}


def case_seed(name):
    return 4242 + sum(map(ord, name))


def make_inputs(name):
    """Initial parameters, states [CALLS, N, S] and target ids [CALLS, N] of a case (what the tests regenerate)."""
    items, n, _ = CASES[name]
    rng = np.random.default_rng(case_seed(name))
    bound = 1.0 / np.sqrt(S)
    w = rng.uniform(-bound, bound, (items, S)).astype(np.float32)
    b = rng.uniform(-bound, bound, items).astype(np.float32)
    states = rng.normal(0.0, 1.0, (CALLS, n, S)).astype(np.float32)
    ids = rng.integers(0, items, (CALLS, n)).astype(np.int64)
    return {"w": w, "b": b, "states": states, "ids": ids}


def input_checksum(inp):
    return np.array([inp["w"].astype(np.float64).sum(), inp["b"].astype(np.float64).sum(),
                     inp["states"].astype(np.float64).sum(), float(inp["ids"].sum())])


def beta_cell_source():
    with open(os.path.join(REFERENCE_ROOT, NOTEBOOK)) as fh:
        nb = json.load(fh)
    for cell in nb["cells"]:
        src = "".join(cell["source"])
        if cell["cell_type"] == "code" and src.lstrip().startswith("class Beta("):
            return src
    raise RuntimeError("class Beta not found in the notebook")


def run_case(name):
    items, n, rows = CASES[name]
    inp = make_inputs(name)
    radam = types.ModuleType("optim")
    radam.RAdam = lambda params, **kw: torch.optim.RAdam(params, decoupled_weight_decay=True, **kw)
    ns = {"nn": torch.nn, "torch": torch, "optim": radam, "num_items": items}
    exec(compile(beta_cell_source(), NOTEBOOK + ":cell3", "exec"), ns)
    beta = ns["Beta"]()
    beta.load_state_dict({"net.0.weight": torch.from_numpy(inp["w"]), "net.0.bias": torch.from_numpy(inp["b"])})
    losses = []
    beta.criterion.register_forward_hook(lambda mod, args, out: losses.append(float(out.detach())))
    out = {"input_checksum": input_checksum(inp), "rows": np.array(rows, np.int64), "ids": inp["ids"],
           "meta": np.array([S, items, n, CALLS, case_seed(name)], np.int64)}
    probs, gw, gb, sw, sb = [], [], [], [], []
    lin = beta.net[0]
    for t in range(CALLS):
        onehot = torch.zeros(n, items)
        onehot[torch.arange(n), torch.from_numpy(inp["ids"][t])] = 1.0
        p = beta(torch.from_numpy(inp["states"][t]), onehot)
        probs.append(p.numpy().copy())
        gw.append(lin.weight.grad[list(rows)].numpy().copy())
        gb.append(lin.bias.grad.numpy().copy())
        if t + 1 in SNAP_AFTER:
            sw.append(lin.weight.detach()[list(rows)].numpy().copy())
            sb.append(lin.bias.detach().numpy().copy())
    out.update(probs=np.stack(probs), loss=np.array(losses), grad_w=np.stack(gw), grad_b=np.stack(gb),
               after_w=np.stack(sw), after_b=np.stack(sb), snap_after=np.array(SNAP_AFTER, np.int64))
    return out


def main():
    torch.set_num_threads(1)
    for name in CASES:
        out = run_case(name)
        path = os.path.join(GOLDEN_DIR, "beta_%s.npz" % name)
        np.savez(path, **out)
        print("wrote", path, "loss", out["loss"])


if __name__ == "__main__":
    main()
