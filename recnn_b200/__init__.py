"""recnn_b200: H100-native implementation of RecNN's DDPG/TD3 update hot path
(gather -> Actor/Critic forward+backward -> losses -> optimizer -> Polyak), behind
RecNN's own Python API.  See DESIGN.md for scope and INTEGRATION.md for drop-in use.
"""
from . import _lib, optim, utils, data, nn, dist

__version__ = "0.1.0"


def install_as_recnn():
    """Register this package under the reference's import names (``recnn``,
    ``recnn.nn``, ``recnn.nn.update``, ``recnn.data``, ``recnn.utils`` ...) so code
    written against awarebayes/RecNN resolves to the H100 path for the hot-path
    symbols.  Raises if the real ``recnn`` is already imported."""
    import sys
    existing = sys.modules.get("recnn")
    if existing is not None and existing is not sys.modules[__name__]:
        raise ImportError("a different 'recnn' package is already imported")
    alias = {
        "recnn": sys.modules[__name__],
        "recnn.nn": nn, "recnn.nn.models": nn.models, "recnn.nn.algo": nn.algo, "recnn.nn.update": nn.update,
        "recnn.nn.update.ddpg": nn.update.ddpg, "recnn.nn.update.td3": nn.update.td3,
        "recnn.nn.update.misc": nn.update.misc, "recnn.nn.update.reinforce": nn.update.reinforce,
        "recnn.data": data, "recnn.data.utils": data.utils, "recnn.data.env": data.env, "recnn.data.db_con": data.db_con,
        "recnn.utils": utils, "recnn.utils.misc": utils.misc, "recnn.optim": optim,
    }
    sys.modules.update(alias)
    return sys.modules[__name__]
