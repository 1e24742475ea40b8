"""Shared helpers: run a seeded update case through a backend and compare the
result with the golden fixtures produced from the real reference
(oracle/make_golden.py)."""
from __future__ import annotations

import os

import numpy as np

from oracle import cases as C
from oracle import recnn_oracle as O

GOLDEN_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
SNAP_AFTER = (1, 2, 11, 12)


def load_golden(name):
    return dict(np.load(os.path.join(GOLDEN_DIR, name)))


def oracle_optimizers(kind, algo):
    mk = (lambda: O.make_optimizer("adam", lr=1e-5)) if kind == "adam" else \
         (lambda: O.make_optimizer("ranger", lr=1e-4, weight_decay=1e-2)) if kind == "ranger" else \
         (lambda: O.make_optimizer("sgd", lr=1e-3, momentum=0.9, weight_decay=1e-3)) if kind == "sgd_momentum" else \
         (lambda: O.make_optimizer("sgd", lr=1e-3))
    names = ("policy_optimizer", "value_optimizer") if algo == "ddpg" else \
            ("policy_optimizer", "value_optimizer1", "value_optimizer2")
    return {n: mk() for n in names}


def run_oracle_case(case, algo, opt_kind, golden=None, inp=None):
    """Same bookkeeping as oracle/make_golden.py:run_update_case, numpy oracle.
    ``inp``: pre-made inputs (C.make_inputs, possibly with edited masks) instead of regenerating them."""
    spec = C.CASES[case] if isinstance(case, str) else case      # a name or a spec dict
    if inp is None:
        inp = C.make_inputs(spec, algo)
    out = {"input_checksums": C.input_checksums(inp)}
    nets = {k: O.copy_net(v) for k, v in inp["nets"].items()}
    opts = oracle_optimizers(opt_kind, algo)
    batch = O.frame_gather(inp["table"], inp["items"], inp["ratings"], inp["sizes"], spec["frame"])
    params = dict(C.DDPG_PARAMS if algo == "ddpg" else C.TD3_PARAMS)
    loss_keys = ("value", "policy") if algo == "ddpg" else ("value1", "value2", "policy")
    losses = {k: [] for k in loss_keys}
    for step in range(spec["steps"]):
        masks = inp["masks"][step]
        if algo == "ddpg":
            loss, dbg = O.ddpg_update(batch, params, nets, opts, masks, step, learn=True)
        else:
            noise = golden["noise.%d" % step] if golden is not None else inp["noise"][step]
            loss, dbg = O.td3_update(batch, params, nets, opts, masks, noise, step, learn=True)
        for k in loss_keys:
            losses[k].append(loss[k])
        done_steps = step + 1
        if done_steps in SNAP_AFTER:
            for name, p in nets.items():
                for k, v in C.net_digest(p).items():
                    out["after%d.%s.%s" % (done_steps, name, k)] = v
        if step == 0 and algo == "ddpg":
            for k, v in C.net_digest(dbg["policy_grads"]).items():
                out["grad_step0.policy_net.%s" % k] = v
        if step == 1 and algo == "ddpg":
            for k, v in C.net_digest(dbg["value_grads"]).items():
                out["grad_step1.value_net.%s" % k] = v
    for k in loss_keys:
        out["loss." + k] = np.asarray(losses[k], dtype=np.float64)
    for name, p in nets.items():
        for k, v in p.items():
            out["final.%s.%s" % (name, k)] = v
    return out


def neutralise_ambiguous_gates(spec, algo, opt_kind, thresh=2e-5, max_iter=8):
    """Inputs of a case whose replayed dropout masks DROP every unit whose ReLU gate is ambiguous.

    ReLU makes the weight gradients discontinuous: a pre-activation within rounding error of 0 may be gated
    either way by two correct fp32 implementations, and each such flip moves that sample's contribution to the
    gradients by O(1/N).  Small golden cases avoid this by seed screening (oracle/find_seeds.py); at BASELINE's
    full size (4096 rows x 256 units x 2 layers x the nets that get a backward x steps = tens of millions of gates)
    no seed is clean.  Here the oracle is run with a log of every KEPT unit with |pre-activation| <= thresh (far
    above the ~1e-6 difference between fp32 GEMM implementations), those units are dropped from the masks (a
    dropped unit outputs 0 and has gradient 0 whatever its gate), and the run is repeated until the log is empty
    (dropping units perturbs later layers / steps, so a few rounds are needed).  Returns (inputs, units dropped,
    rounds).  With these inputs every gate decision is unambiguous and the tight parity bar applies to EVERY
    weight at full size."""
    inp = C.make_inputs(spec, algo)
    total = 0
    for it in range(max_iter):
        O.GATE_LOG.update(on=True, thresh=float(thresh), hits=[])
        try:
            run_oracle_case(spec, algo, opt_kind, inp=inp)
        finally:
            O.GATE_LOG["on"] = False
        hits, O.GATE_LOG["hits"] = O.GATE_LOG["hits"], []
        if not hits:
            return inp, total, it
        for mask, rows, cols in hits:
            mask[rows, cols] = 0
            total += int(rows.size)
    raise AssertionError("ambiguous gates remain after %d rounds" % max_iter)


def assert_tight_parity(got, want, init_nets, loss_rtol=1e-5, rtol=1e-5, floor_frac=1e-2, delta_rtol=2e-3,
                        outliers=0, outlier_abs=0.0):
    """The golden bar on EVERY element of every final weight (a run with no ambiguous ReLU gate, see
    neutralise_ambiguous_gates).  ``got`` / ``want``: run_cuda_case / run_oracle_case outputs; ``init_nets``: the
    nets the run started from (C.make_inputs(...)["nets"]).

    Losses: |got-want| <= loss_rtol*(|want| + 0.1).  Weights: |got-want| <= rtol*(|want| + floor_frac*max|tensor|).
    Weight changes since init: within delta_rtol of the tensor's largest change, beyond 2 ulp of its largest weight
    (differences below that are rounding of the stored weight, not signal).  A tensor that does not move must stay
    bit-identical.

    ``outliers``: elements per tensor that may miss the weight / change bars, each by at most ``outlier_abs``.  Only
    for Adam, whose g / (|g| + eps) turns the fp32 rounding of a gradient that nearly cancels into an lr-sized
    difference of that one element.  Returns the largest error found on each bar (outliers excluded), the largest
    outlier count of a tensor and the number of tensors whose change was checked."""
    rep = {"loss": 0.0, "weight": 0.0, "delta": 0.0, "outliers": 0, "checked": 0}
    for k in (k for k in want if k.startswith("loss.")):
        err = float(np.max(np.abs(got[k] - want[k]) / (np.abs(want[k]) + 0.1)))
        rep["loss"] = max(rep["loss"], err)
        assert err <= loss_rtol, (k, err, got[k], want[k])
    for k in (k for k in want if k.startswith("final.")):
        _, name, tensor = k.split(".")
        init = init_nets[name][tensor].astype(np.float64)
        w_want, w_got = want[k].astype(np.float64), got[k].astype(np.float64)
        wmax = np.max(np.abs(w_want))
        rel = np.abs(w_got - w_want) / (np.abs(w_want) + floor_frac * wmax)
        d_want, d_got = w_want - init, w_got - init
        scale = np.max(np.abs(d_want))
        if scale == 0.0:                       # e.g. TD3's target policy is never updated (td3.py:136-141)
            assert np.array_equal(got[k], want[k]), k
            continue
        ulp2 = 2.0 * 1.1920929e-07 * wmax
        excess = np.maximum(np.abs(d_got - d_want) - ulp2, 0.0) / scale
        bad = (rel > rtol) | (excess > delta_rtol)
        n_bad = int(bad.sum())
        assert n_bad <= outliers, (k, n_bad, float(rel.max()), float(excess.max()))
        if n_bad:
            assert np.max(np.abs(w_got - w_want)[bad]) <= outlier_abs, (k, np.max(np.abs(w_got - w_want)[bad]))
        rep["weight"] = max(rep["weight"], float(np.max(rel[~bad])))
        rep["delta"] = max(rep["delta"], float(np.max(excess[~bad])))
        rep["outliers"] = max(rep["outliers"], n_bad)
        rep["checked"] += 1
    return rep


def assert_oracle_bar(got, want, init_nets, rtol=1e-5):
    """The bar of the optimizers without golden fixtures (Ranger, SGD with momentum) against run_oracle_case: losses
    within 1e-5 of |want| + 0.1; every final weight within ``rtol`` relative (floor: 1e-2 of the tensor's largest weight);
    every weight change within 2e-3 of the tensor's largest change, beyond 2 ulp of its largest weight.  A tensor that
    does not move must stay bit-identical.  Returns the largest error found on each bar."""
    rep = {"loss": 0.0, "weight": 0.0, "delta": 0.0}
    for k in (k for k in want if k.startswith("loss.")):
        err = float(np.max(np.abs(got[k] - want[k]) / (np.abs(want[k]) + 0.1)))
        rep["loss"] = max(rep["loss"], err)
        assert err <= 1e-5, (k, err)
    for k in (k for k in want if k.startswith("final.")):
        _, name, tensor = k.split(".")
        w = want[k].astype(np.float64)
        wmax = np.max(np.abs(w))
        err = float(np.max(np.abs(got[k] - w) / (np.abs(w) + 1e-2 * wmax)))
        rep["weight"] = max(rep["weight"], err)
        assert err <= rtol, (k, err)
        d_want = w - init_nets[name][tensor]
        scale = np.max(np.abs(d_want))
        if scale == 0:
            assert np.array_equal(got[k], want[k]), k
            continue
        ulp2 = 2.0 * 1.1920929e-07 * wmax
        excess = float(np.max(np.maximum(np.abs((got[k] - init_nets[name][tensor]) - d_want) - ulp2, 0)) / scale)
        rep["delta"] = max(rep["delta"], excess)
        assert excess <= 2e-3, (k, excess)
    return rep


def rel_err(got, want, floor):
    got = np.asarray(got, dtype=np.float64)
    want = np.asarray(want, dtype=np.float64)
    return float(np.max(np.abs(got - want) / (np.abs(want) + floor))) if got.size else 0.0


def compare_with_golden(got: dict, gold: dict, rtol=1e-5, floor_frac=1e-2, delta_rtol=2e-3,
                        grad_rtol=1e-4, check_grads=True, loss_floor=0.1):
    """The north-star bar: losses and every updated weight within 1e-5 relative.

    Weights: |got-want| <= rtol*(|want| + floor_frac*max|tensor|).  The reference
    defines no floor for near-zero weights (SURVEY.md 8c); floor_frac=1e-2 makes
    the absolute part 1e-7*max|tensor| ~ one fp32 ulp of the tensor's largest
    weight, which is what two fp32 BLAS builds already differ by.
    Losses: |got-want| <= rtol*(|want| + loss_floor).  The policy loss is a
    signed mean of Q-values of magnitude O(1..10) that nearly cancels, so a pure
    relative bound is below one fp32 ulp of the summands (torch/MKL and
    numpy/OpenBLAS differ by 3e-5 relative there); loss_floor=0.1 makes the
    absolute part 1e-6 ~ 1 ulp at |Q| ~ 10 = max_value.
    Deltas: with lr=1e-5 the 1e-5 bar alone would be met by not training at
    all, so the *change* of each tensor since init must also agree to
    ``delta_rtol`` of its largest change (differences below 2 ulp of the
    tensor's largest weight are rounding, not signal, and are accepted).
    Grads: within ``grad_rtol`` of the largest gradient entry of the tensor."""
    np.testing.assert_allclose(got["input_checksums"], gold["input_checksums"], rtol=1e-12,
                               err_msg="regenerated inputs differ from the golden run's inputs")
    assert float(gold["gate_margin"]) > C.GATE_GUARD, "golden case has an ambiguous ReLU gate"
    report = {}
    for key in sorted(k for k in gold if k.startswith("loss.")):
        e = rel_err(got[key], gold[key], loss_floor)
        report[key] = e
        assert e <= rtol, "%s: rel err %.3g > %.3g\n got  %s\n want %s" % (key, e, rtol, got[key], gold[key])
    for key in sorted(gold):
        if not key.startswith("after") or not key.endswith(".sample"):
            continue
        wmax = float(np.max(np.abs(gold[key])))
        e = rel_err(got[key], gold[key], floor_frac * wmax)
        report[key] = e
        assert e <= rtol, "%s: rel err %.3g > %.3g" % (key, e, rtol)
        _, name, tensor, _ = key.split(".")
        init = gold["init.%s.%s.sample" % (name, tensor)].astype(np.float64)
        d_got = got[key].astype(np.float64) - init
        d_want = gold[key].astype(np.float64) - init
        scale = np.max(np.abs(d_want))
        err = float(np.max(np.abs(d_got - d_want)))
        ulp2 = 2.0 * 1.1920929e-07 * wmax
        de = err / scale if scale > 0 else (0.0 if err == 0 else np.inf)
        report[key + ".delta"] = de
        assert de <= delta_rtol or err <= ulp2, \
            "%s: delta err %.3g > %.3g (scale %.3g, abs %.3g)" % (key, de, delta_rtol, scale, err)
    if check_grads:
        for key in sorted(k for k in gold if k.startswith("grad_") and k.endswith(".sample")):
            if key not in got:
                continue
            scale = np.max(np.abs(gold[key])) + 1e-30
            e = float(np.max(np.abs(got[key].astype(np.float64) - gold[key])) / scale)
            report[key] = e
            assert e <= grad_rtol, "%s: grad err %.3g > %.3g of max |g|" % (key, e, grad_rtol)
    return report
