"""Flat parameter / gradient arenas behind Actor and Critic.

The CUDA kernels address a net as ONE fp32 buffer in ``nn.Module.parameters()`` order
(include/recnn_b200.h, "net") whose matrix rows are padded to 16-byte multiples so that
every weight is a legal TMA tensor (linear1.weight of the Actor: [256, 1290] with row
pitch 1292).  The modules keep ordinary ``nn.Parameter`` objects -- ``state_dict`` keys
linear{1,2,3}.{weight,bias} stay loadable (examples/streamlit_demo.py:152-160 in the
reference) and external torch optimizers keep working -- but their storage is a (possibly
strided) view into the arena; pad elements are zero and stay zero.
``module.to(device)``, ``load_state_dict`` into fresh tensors or
``zero_grad(set_to_none=True)`` can break that aliasing, so every kernel entry
re-validates it (a few pointer compares) and rebuilds the arena if needed.
"""
from __future__ import annotations

import ctypes

import torch

from .. import _lib


def _is_discrete(module):
    """Two-layer DiscreteActor (recnn/nn/models.py:76-99): linear1, linear2 and nothing else."""
    return not hasattr(module, "linear3")


def _is_beta(module):
    """The Top-K notebook's behaviour policy (nn.Beta): one nn.Linear in ``module.net[0]``."""
    return getattr(module, "_recnn_beta", False)


def _params(module):
    if _is_beta(module):
        return [module.net[0].weight, module.net[0].bias]
    ps = [module.linear1.weight, module.linear1.bias, module.linear2.weight, module.linear2.bias]
    if not _is_discrete(module):
        ps += [module.linear3.weight, module.linear3.bias]
    return ps


def discrete_dims(module):
    return _lib.DiscreteDims(module.linear1.in_features, module.linear1.out_features, module.linear2.out_features, 0)


def net_layout(module):
    """(offsets[6], pitches[3], count) of this module's arena, from the C library (4 offsets / 2 pitches for the
    two-layer DiscreteActor, 2 offsets / 1 pitch for nn.Beta)."""
    if _is_beta(module):
        buf = (ctypes.c_int64 * 4)()
        _lib.check(_lib.lib().recnn_beta_layout(module.dims, buf))
        v = list(buf)
        return v[0:2], v[2:3], v[3]
    if _is_discrete(module):
        buf = (ctypes.c_int64 * 7)()
        _lib.check(_lib.lib().recnn_discrete_layout(discrete_dims(module), buf))
        v = list(buf)
        return v[0:4], v[4:6], v[6]
    s = module.linear1.in_features
    h = module.linear1.out_features
    out = module.linear3.out_features
    is_critic = out == 1 and hasattr(module, "_action_dim")
    if is_critic:
        a = module._action_dim
        dims = _lib.Dims(s - a, a, h, 0)
    else:
        is_critic = False
        dims = _lib.Dims(s, out, h, 0)
    buf = (ctypes.c_int64 * 10)()
    _lib.check(_lib.lib().recnn_net_layout(dims, int(is_critic), buf))
    v = list(buf)
    return v[0:6], v[6:9], v[9]


def _views(flat, module):
    offs, lds, _ = net_layout(module)
    ps = _params(module)
    out = []
    for i, p in enumerate(ps):
        if p.dim() == 2:
            rows, cols = p.shape
            ld = lds[i // 2]
            out.append(flat[offs[i]: offs[i] + rows * ld].view(rows, ld)[:, :cols])
        else:
            out.append(flat[offs[i]: offs[i] + p.numel()])
    return out


def _aliases(flat, module, tensors):
    if flat is None:
        return False
    for view, t in zip(_views(flat, module), tensors):
        if t is None or t.device != flat.device or t.dtype != torch.float32:
            return False
        if t.data_ptr() != view.data_ptr() or t.stride() != view.stride() or t.shape != view.shape:
            return False
    return True


def param_arena(module) -> torch.Tensor:
    """Flat fp32 arena holding all parameters of ``module`` (rebuilt if aliasing broke)."""
    ps = _params(module)
    flat = getattr(module, "_recnn_flat", None)
    if flat is not None and flat.device == ps[0].device and _aliases(flat, module, [p.data for p in ps]):
        return flat
    dev = ps[0].device
    _, _, count = net_layout(module)
    flat = torch.zeros(count, dtype=torch.float32, device=dev)
    with torch.no_grad():
        for p, view in zip(ps, _views(flat, module)):
            view.copy_(p.data.to(device=dev, dtype=torch.float32))
            p.data = view
    object.__setattr__(module, "_recnn_flat", flat)
    object.__setattr__(module, "_recnn_flat_grad", None)
    return flat


def grad_arena(module) -> torch.Tensor:
    """Flat fp32 gradient arena (same geometry); ``p.grad`` of every parameter is a view into it."""
    ps = _params(module)
    flat = param_arena(module)
    g = getattr(module, "_recnn_flat_grad", None)
    if g is None or g.device != flat.device or g.numel() != flat.numel():
        g = torch.zeros_like(flat)
        object.__setattr__(module, "_recnn_flat_grad", g)
    if not _aliases(g, module, [p.grad for p in ps]):
        for p, view in zip(ps, _views(g, module)):
            p.grad = view
    return g
