"""Run the seeded cases of oracle/cases.py through the CUDA path (public Python API ->
C ABI) and digest the result the same way oracle/make_golden.py does."""
from __future__ import annotations

import numpy as np
import torch

import recnn_b200
from oracle import cases as C
from oracle import recnn_oracle as O

SNAP_AFTER = (1, 2, 11, 12)


def load_net(module, p, device):
    with torch.no_grad():
        for lin, w, b in ((module.linear1, "w1", "b1"), (module.linear2, "w2", "b2"), (module.linear3, "w3", "b3")):
            lin.weight.copy_(torch.from_numpy(p[w]))
            lin.bias.copy_(torch.from_numpy(p[b]))
    return module.to(device)


def dump_net(module):
    ps = [module.linear1.weight, module.linear1.bias, module.linear2.weight, module.linear2.bias,
          module.linear3.weight, module.linear3.bias]
    return dict(zip(O.PARAM_ORDER, [q.detach().cpu().numpy().copy() for q in ps]))


def dump_grad(module):
    ps = [module.linear1.weight, module.linear1.bias, module.linear2.weight, module.linear2.bias,
          module.linear3.weight, module.linear3.bias]
    return dict(zip(O.PARAM_ORDER, [q.grad.detach().cpu().numpy().copy() for q in ps]))


def build_nets(spec, inp, device):
    s_dim, a_dim, h = C.dims(spec)
    nets = {}
    for name, p in inp["nets"].items():
        if "policy" in name:
            m = recnn_b200.nn.Actor(s_dim, a_dim, h, spec["actor_init_w"])
        else:
            m = recnn_b200.nn.Critic(s_dim, a_dim, h, spec["critic_init_w"])
        load_net(m, p, device)
        m.eval() if "target" in name else m.train()
        nets[name] = m
    return nets


def build_optimizers(kind, nets, algo, external=False):
    def mk(net):
        if external:
            return torch.optim.Adam(net.parameters(), lr=1e-5) if kind == "adam" else \
                torch.optim.SGD(net.parameters(), lr=1e-3)
        if kind == "ranger":
            return recnn_b200.optim.Ranger(net.parameters(), lr=1e-4, weight_decay=1e-2)
        if kind == "sgd_momentum":
            return recnn_b200.optim.SGD(net.parameters(), lr=1e-3, momentum=0.9, weight_decay=1e-3)
        return recnn_b200.optim.Adam(net.parameters(), lr=1e-5) if kind == "adam" else \
            recnn_b200.optim.SGD(net.parameters(), lr=1e-3)
    names = {"policy_optimizer": "policy_net"}
    if algo == "ddpg":
        names["value_optimizer"] = "value_net"
    else:
        names["value_optimizer1"] = "value_net1"
        names["value_optimizer2"] = "value_net2"
    return {k: mk(nets[v]) for k, v in names.items()}


def run_cuda_case(case, algo, opt_kind, golden=None, form="dense", external=False, device="cuda:0",
                  shard=None, inp=None, comm=None, on_step=None):
    """shard=(rank, world): this process handles rows [lo, hi) of every minibatch (data parallel).
    ``inp``: pre-made inputs (C.make_inputs, possibly with edited masks) instead of regenerating them.
    ``comm``: callable nets -> peer communicator (an object with ``.ptr``), attached before the first update so the
    step runs its gradient all-reduce kernels through it.  ``on_step(step, nets, opts, loss)``: called after each
    update."""
    spec = C.CASES[case] if isinstance(case, str) else case      # a name or a spec dict
    if inp is None:
        inp = C.make_inputs(spec, algo)
    dev = torch.device(device)
    lo, hi = (0, spec["n_rows"]) if shard is None else recnn_b200.dist.shard_rows(spec["n_rows"], *shard)
    out = {"input_checksums": C.input_checksums(inp)}
    nets = build_nets(spec, inp, dev)
    opts = build_optimizers(opt_kind, nets, algo, external)
    if shard is not None:
        recnn_b200.dist.enable_data_parallel(nets)
    if comm is not None:           # read by get_engine when it creates the engine, i.e. on the first update
        nets["policy_net"].__dict__["_recnn_dp"] = (None, 1, comm(nets))
    params = dict(C.DDPG_PARAMS if algo == "ddpg" else C.TD3_PARAMS)
    table = torch.from_numpy(inp["table"]).to(dev)
    ref = O.frame_gather(inp["table"], inp["items"], inp["ratings"], inp["sizes"], spec["frame"])
    if form == "dense":
        base = {k: torch.from_numpy(v[lo:hi]) for k, v in ref.items()}   # host tensors, like the reference's loader
    elif shard is None:
        base = {"items": torch.from_numpy(inp["items"]), "ratings": torch.from_numpy(inp["ratings"]),
                "sizes": torch.from_numpy(inp["sizes"]), "table": table}
    else:                        # `done` is a prefix computation over the whole batch: sliced after the fact
        base = {"items": torch.from_numpy(inp["items"][lo:hi]), "ratings": torch.from_numpy(inp["ratings"][lo:hi]),
                "done": torch.from_numpy(ref["done"][lo:hi]), "table": table}
    update = recnn_b200.nn.ddpg_update if algo == "ddpg" else recnn_b200.nn.td3_update
    loss_keys = ("value", "policy") if algo == "ddpg" else ("value1", "value2", "policy")
    losses = {k: [] for k in loss_keys}
    for step in range(spec["steps"]):
        batch = dict(base)
        batch["dropout_masks"] = [torch.from_numpy(np.ascontiguousarray(m[lo:hi])) for m in inp["masks"][step]]
        if algo == "td3":
            nz = golden["noise.%d" % step] if golden is not None else inp["noise"][step]
            batch["noise"] = torch.from_numpy(np.ascontiguousarray(nz[lo:hi]))
        loss = update(batch, params, nets, opts, dev, {}, recnn_b200.utils.DummyWriter(), learn=True, step=step)
        assert loss["step"] == step
        if on_step is not None:
            on_step(step, nets, opts, loss)
        for k in loss_keys:
            losses[k].append(loss[k])
        done_steps = step + 1
        if done_steps in SNAP_AFTER:
            for name, m in nets.items():
                for k, v in C.net_digest(dump_net(m)).items():
                    out["after%d.%s.%s" % (done_steps, name, k)] = v
        if step == 0:
            for k, v in C.net_digest(dump_grad(nets["policy_net"])).items():
                out["grad_step0.policy_net.%s" % k] = v
        if step == 1:
            crit = "value_net" if algo == "ddpg" else "value_net1"
            for k, v in C.net_digest(dump_grad(nets[crit])).items():
                out["grad_step1.%s.%s" % (crit, k)] = v
    for k in loss_keys:
        out["loss." + k] = np.asarray(losses[k], dtype=np.float64)
    for name, m in nets.items():
        for k, v in dump_net(m).items():
            out["final.%s.%s" % (name, k)] = v
    out["_nets"] = nets
    out["_opts"] = opts
    return out
