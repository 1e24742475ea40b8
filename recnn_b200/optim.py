"""Built-in optimizers whose step is fused into the device update step.

``recnn_b200.optim.Adam`` / ``SGD`` follow torch.optim.Adam / SGD (torch 2.11
single-tensor semantics: lerp_ for exp_avg, bias corrections formed in double,
L2-style weight_decay) but keep their state as flat arenas next to the net's
parameter arena, so the update functions can run the optimizer as part of the
same CUDA graph.  They are torch.optim.Optimizer subclasses: ``zero_grad``,
``param_groups`` (lr can be edited between steps) behave as usual, ``state_dict`` /
``load_state_dict`` carry the flat moment arenas and the step count (``recnn_arenas``), and ``step()`` may also be called on its own.

Any other torch optimizer passed through the reference's ``optimizer`` dict is
honoured too (the step is then split at the points where gradients are
complete and ``optimizer.step()`` is called in between); the reference's default
``torch_optimizer.Ranger`` is not reproducible here (SURVEY.md fact 4).
"""
from __future__ import annotations

import torch

from . import _lib


class _ArenaOptimizer(torch.optim.Optimizer):
    _recnn_kind = _lib.OPT_EXTERNAL

    def __init__(self, params, defaults):
        super().__init__(params, defaults)
        if len(self.param_groups) != 1:
            raise ValueError("recnn_b200 optimizers take a single parameter group (one net)")
        self._m = self._v = self._t = self._slow = None
        self._module = None

    # -- binding to a net -------------------------------------------------------
    def bind(self, module):
        """Associate with the Actor/Critic whose parameters this optimizer owns."""
        from .nn.arena import _params
        mine = [id(p) for p in self.param_groups[0]["params"]]
        theirs = [id(p) for p in _params(module)]
        if mine != theirs:
            raise ValueError("optimizer parameters are not exactly this net's parameters()")
        self._module = module
        return self

    def _state_arenas(self, flat):
        if self._t is None:
            self._t = torch.zeros(1, dtype=torch.int32, device=flat.device)
            self._m = torch.zeros_like(flat)
            self._v = (torch.zeros_like(flat) if self._recnn_kind in (_lib.OPT_ADAM, _lib.OPT_RANGER, _lib.OPT_RADAM)
                       else None)
            self._slow = torch.zeros_like(flat) if self._recnn_kind == _lib.OPT_RANGER else None
        elif self._t.device != flat.device or self._m.numel() != flat.numel():
            if self._m.numel() != flat.numel():
                raise _lib.RecnnError("optimizer state (%d elements) does not match the net's arena (%d)"
                                      % (self._m.numel(), flat.numel()))
            # the net moved (Algo.to(device)): the moments and the step count move with it
            self._t = self._t.to(flat.device)
            self._m = self._m.to(flat.device)
            self._v = None if self._v is None else self._v.to(flat.device)
            self._slow = None if self._slow is None else self._slow.to(flat.device)
        return self._m, self._v, self._t

    # -- checkpointing: the moments / step count live in flat arenas, not in self.state -----------
    def state_dict(self):
        """torch's layout plus ``recnn_arenas``: the flat moment arenas (geometry of the net's parameter
        arena, pads included) and the step count, so a resumed run continues the bias correction."""
        sd = super().state_dict()
        if self._t is not None:
            sd["recnn_arenas"] = {"m": self._m.detach().cpu().clone(),
                                  "v": None if self._v is None else self._v.detach().cpu().clone(),
                                  "slow": None if self._slow is None else self._slow.detach().cpu().clone(),
                                  "t": int(self._t.item())}
        return sd

    def load_state_dict(self, state_dict):
        state_dict = dict(state_dict)
        arenas = state_dict.pop("recnn_arenas", None)
        super().load_state_dict(state_dict)
        if arenas is None:
            self._m = self._v = self._t = self._slow = None
            return
        dev = self.param_groups[0]["params"][0].device
        self._m = arenas["m"].to(dev).clone()
        self._v = None if arenas["v"] is None else arenas["v"].to(dev).clone()
        self._slow = None if arenas.get("slow") is None else arenas["slow"].to(dev).clone()
        self._t = torch.full((1,), int(arenas["t"]), dtype=torch.int32, device=dev)

    def c_optim(self) -> _lib.Optim:
        raise NotImplementedError

    def c_net(self, module=None) -> _lib.Net:
        from .nn.arena import param_arena, grad_arena
        module = module or self._module
        if module is None:
            raise _lib.RecnnError("optimizer is not bound to a net; call .bind(net) or pass it through an update function")
        flat = param_arena(module)
        g = grad_arena(module)
        m, v, t = self._state_arenas(flat)
        return _lib.Net(flat.data_ptr(), g.data_ptr(), _lib.ptr(m), _lib.ptr(v), t.data_ptr(), _lib.ptr(self._slow))

    @torch.no_grad()
    def step(self, closure=None):
        if closure is not None:
            raise ValueError("closures are not supported")
        from .nn.arena import param_arena
        if self._module is None:
            raise _lib.RecnnError("optimizer is not bound to a net; call .bind(net) first")
        flat = param_arena(self._module)
        net = self.c_net()
        opt = self.c_optim()
        with torch.cuda.device(flat.device):
            _lib.check(_lib.lib().recnn_optimizer_step(opt, net, flat.numel(), None, _lib.stream_ptr(flat.device)))

    def steps_taken(self) -> int:
        return 0 if self._t is None else int(self._t.item())


class Adam(_ArenaOptimizer):
    _recnn_kind = _lib.OPT_ADAM

    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0):
        super().__init__(params, dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay))

    def c_optim(self):
        g = self.param_groups[0]
        return _lib.Optim(_lib.OPT_ADAM, 0, float(g["lr"]), float(g["betas"][0]), float(g["betas"][1]),
                          float(g["eps"]), float(g["weight_decay"]), 0.0, 0.0, 0.0)


class SGD(_ArenaOptimizer):
    _recnn_kind = _lib.OPT_SGD

    def __init__(self, params, lr=1e-3, momentum=0.0, weight_decay=0.0):
        super().__init__(params, dict(lr=lr, momentum=momentum, weight_decay=weight_decay))

    def c_optim(self):
        g = self.param_groups[0]
        return _lib.Optim(_lib.OPT_SGD, 0, float(g["lr"]), 0.0, 0.0, 0.0, float(g["weight_decay"]),
                          float(g["momentum"]), 0.0, 0.0)


class Ranger(_ArenaOptimizer):
    """torch_optimizer.Ranger (RAdam + Lookahead), the optimizer recnn.nn.DDPG / TD3 build by default
    (recnn/nn/algo.py:84-89: ``Ranger(params, lr=..., weight_decay=...)``), with the package's signature and
    defaults.  torch_optimizer is not vendored in the reference and not installed here; this follows the published
    algorithm (rectified Adam with the N_sma_threshhold switch, Lookahead with slow weights every k steps) and its
    bit-level parity with the package is UNPINNED -- see DESIGN.md section 2."""
    _recnn_kind = _lib.OPT_RANGER

    def __init__(self, params, lr=1e-3, alpha=0.5, k=6, N_sma_threshhold=5, betas=(0.95, 0.999), eps=1e-5,
                 weight_decay=0):
        if not 0.0 <= alpha <= 1.0:
            raise ValueError("Invalid slow update rate: %r" % alpha)
        if not 1 <= k:
            raise ValueError("Invalid lookahead steps: %r" % k)
        super().__init__(params, dict(lr=lr, alpha=alpha, k=k, N_sma_threshhold=N_sma_threshhold, betas=betas,
                                      eps=eps, weight_decay=weight_decay))

    def c_optim(self):
        g = self.param_groups[0]
        return _lib.Optim(_lib.OPT_RANGER, int(g["k"]), float(g["lr"]), float(g["betas"][0]), float(g["betas"][1]),
                          float(g["eps"]), float(g["weight_decay"]), 0.0, float(g["alpha"]),
                          float(g["N_sma_threshhold"]))


class RAdam(_ArenaOptimizer):
    """torch_optimizer.RAdam, the optimizer of the Top-K notebook's behaviour policy (``optim.RAdam(lr=1e-5,
    weight_decay=1e-5)``), with the package's signature and defaults: rectified Adam switched on from N_sma >= 5 and
    decoupled weight decay -- Ranger's RAdam half without Lookahead.  Pinned against
    ``torch.optim.RAdam(decoupled_weight_decay=True)``; parity with the package itself is UNPINNED, as for Ranger
    (DESIGN.md section 2)."""
    _recnn_kind = _lib.OPT_RADAM

    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0):
        super().__init__(params, dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay))

    def c_optim(self):
        g = self.param_groups[0]
        return _lib.Optim(_lib.OPT_RADAM, 0, float(g["lr"]), float(g["betas"][0]), float(g["betas"][1]),
                          float(g["eps"]), float(g["weight_decay"]), 0.0, 0.0, 5.0)
