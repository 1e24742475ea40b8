"""Drop-in for recnn.nn.update.reinforce (recnn/nn/update/reinforce.py:10-129): ChooseREINFORCE and reinforce_update.

The policy loss and its gradient are ONE device call (recnn_reinforce_policy_grad_chunked: recomputed forward,
closed-form d loss / d logits, three tensor-core GEMMs; over item chunks when the [rows, num_items] logits would exceed
_LOGITS_BUDGET_BYTES) over the rows ``DiscreteActor`` saved since the last policy update; the
optimizer step is the fused arena kernel (recnn_b200.optim) or any torch optimizer stepping the aliased ``.grad``
views.  The critic half is the DDPG critic step (value_update) fed with the target policy's probabilities, or -- when
``batch["action"]`` holds integer item ids -- the item-id critic step of _ids.py, which never forms a [N, num_items]
matrix.
"""
from __future__ import annotations

import gc

import torch

from ... import _lib
from ... import utils
from ...utils.misc import DummyWriter
from ..arena import param_arena, grad_arena
from .misc import value_update
from . import _ids

# Largest logits buffer ([rows, chunk] fp32) one policy update may hold.  Below it the whole [rows, num_items] matrix
# is kept (one pass); above it the items are visited in chunks and the logits are computed twice.
_LOGITS_BUDGET_BYTES = 1 << 30


def _chunk_items(rows, num_items):
    """Item chunk width of the policy gradient over ``rows`` saved rows: every item at once when their logits fit in
    _LOGITS_BUDGET_BYTES, otherwise the widest multiple of 128 that fits (at least 128)."""
    if rows * num_items * 4 <= _LOGITS_BUDGET_BYTES:
        return num_items
    chunk = max(128, _LOGITS_BUDGET_BYTES // (rows * 4) // 128 * 128)
    return min(chunk, num_items)


def _policy_loss(policy, returns, method):
    """Loss (0-dim tensor) of ``method`` over policy._saved; the gradient of every parameter lands in the policy's
    gradient arena (= ``p.grad`` of its parameters), overwriting what was there (zero_grad + backward)."""
    saved = policy._saved
    if not saved:
        raise RuntimeError("no saved actions: select_action was not called since the last policy update")
    if len(returns) != len(saved):
        raise ValueError("%d returns for %d saved env steps" % (len(returns), len(saved)))
    flat = param_arena(policy)
    dev = flat.device
    if dev.type != "cuda":
        raise _lib.RecnnError("recnn_b200 nets run on CUDA only (policy is on %s)" % dev)
    grads = grad_arena(policy)
    state = torch.cat([r["state"] for r in saved], 0).contiguous()
    action = torch.cat([r["action"] for r in saved], 0).contiguous()
    beta_lp = None
    if method != _lib.REINFORCE_BASIC:
        if any(r["beta_log_prob"] is None for r in saved):
            raise RuntimeError("the corrected REINFORCE losses need select_action to be one of the *_with_correction "
                               "variants (no behaviour-policy log-probs were saved)")
        beta_lp = torch.cat([r["beta_log_prob"] for r in saved], 0).contiguous()
    rows = torch.tensor([r["state"].shape[0] for r in saved])
    ret_rows = torch.repeat_interleave(torch.as_tensor(returns, dtype=torch.float32).cpu(), rows).to(dev, non_blocking=True)
    n = state.shape[0]
    d = policy.dims
    L = _lib.lib()
    chunk = _chunk_items(n, d.num_items)
    scratch = torch.empty(L.recnn_reinforce_scratch_floats(d, n, chunk), device=dev, dtype=torch.float32)
    out = torch.zeros(3, device=dev, dtype=torch.float32)
    ks = {r.get("K") for r in saved if r.get("K") is not None}
    if len(ks) > 1:
        raise ValueError("select_action was called with different K since the last policy update: %s" % sorted(ks))
    K = ks.pop() if ks else 1
    vp = policy.__dict__.get("_recnn_vp")
    with torch.cuda.device(dev):
        if vp is None:
            _lib.check(L.recnn_reinforce_policy_grad_chunked(
                d, flat.data_ptr(), grads.data_ptr(), state.data_ptr(), action.data_ptr(), _lib.ptr(beta_lp),
                ret_rows.data_ptr(), n, method, K, chunk, out.data_ptr(), scratch.data_ptr(), _lib.stream_ptr(dev)))
        else:
            # vocabulary-parallel: row statistics of the local items, all-gather, local dW2 / db2 and this rank's
            # share of the layer-1 gradient, all-reduce of the layer-1 block
            shard = vp.shard()
            rec = torch.empty(L.recnn_vocab_record_floats(n), device=dev, dtype=torch.float32)
            _lib.check(L.recnn_reinforce_shard_stats(d, shard, flat.data_ptr(), state.data_ptr(), action.data_ptr(), n,
                                                     chunk, rec.data_ptr(), scratch.data_ptr(), _lib.stream_ptr(dev)))
            gathered = vp.all_gather(rec)
            _lib.check(L.recnn_reinforce_shard_grad(
                d, shard, flat.data_ptr(), grads.data_ptr(), state.data_ptr(), action.data_ptr(), _lib.ptr(beta_lp),
                ret_rows.data_ptr(), n, method, K, chunk, gathered.data_ptr(), out.data_ptr(), scratch.data_ptr(),
                _lib.stream_ptr(dev)))
            from ...dist import layer1_floats
            vp.all_reduce(grads[:layer1_floats(d)])
    flags = out.view(torch.int32)[1:].tolist()
    if flags[1] != 0:
        raise RuntimeError("the ranks disagree on the vocabulary shard plan or on the saved rows")
    if flags[0] != 0:
        raise IndexError("saved action index out of range for the policy's output layer")
    return out[0].clone()


class ChooseREINFORCE:
    def __init__(self, method=None):
        if method is None:
            method = ChooseREINFORCE.basic_reinforce
        self.method = method

    @staticmethod
    def basic_reinforce(policy, returns, *args, **kwargs):
        """sum over saved steps and rows of -log pi(a) R   (reinforce.py:16-22)"""
        return _policy_loss(policy, returns, _lib.REINFORCE_BASIC)

    @staticmethod
    def reinforce_with_correction(policy, returns, *args, **kwargs):
        """... of (pi(a)/beta(a)) (-log pi(a)) R   (reinforce.py:24-33)"""
        return _policy_loss(policy, returns, _lib.REINFORCE_CORRECTED)

    @staticmethod
    def reinforce_with_TopK_correction(policy, returns, *args, **kwargs):
        """... of lambda_K (pi(a)/beta(a)) (-log pi(a)) R, lambda_K = K (1 - pi(a))^(K-1)   (reinforce.py:35-44)"""
        return _policy_loss(policy, returns, _lib.REINFORCE_TOPK)

    _BUILT_IN = ("basic_reinforce", "reinforce_with_correction", "reinforce_with_TopK_correction")

    def __call__(self, policy, optimizer, learn=True):
        if getattr(self.method, "__name__", None) not in self._BUILT_IN or \
                getattr(ChooseREINFORCE, self.method.__name__) is not self.method:
            raise TypeError("recnn_b200 computes the REINFORCE gradient in closed form for the three built-in methods; "
                            "a custom method would need the autograd graph the reference keeps in saved_log_probs")
        # discounted returns over the saved env steps, normalised (reinforce.py:44-52; the discount is the literal 0.99)
        R = 0
        returns = []
        rewards = [r.detach().float().cpu() if torch.is_tensor(r) else torch.tensor(float(r)) for r in policy.rewards]
        for r in rewards[::-1]:
            R = r + 0.99 * R
            returns.insert(0, R)
        returns = torch.tensor(returns)
        returns = (returns - returns.mean()) / (returns.std() + 0.0001)

        policy_loss = self.method(policy, returns)

        if learn:
            # zero_grad + backward happened inside the method (the gradient arena was overwritten)
            from ... import optim as _optim
            if isinstance(optimizer, _optim._ArenaOptimizer) and optimizer._module is not policy:
                optimizer.bind(policy)
            optimizer.step()

        policy.gc()
        gc.collect()
        return policy_loss


def reinforce_update(batch, params, nets, optimizer, device=torch.device("cpu"), debug=None,
                     writer=DummyWriter(), learn=True, step=-1):
    """Same signature, side effects and return value as the reference (reinforce.py:68-129): returns the losses dict
    on policy steps (step % policy_step == 0 and step > 0) and None otherwise.

    With nets sharded over the item vocabulary (recnn_b200.dist.enable_vocab_parallel on the agent) the batch action
    must be item ids: the reward line feeds the critic the policy's column block (action terms all-reduced) and the
    critic step runs vocabulary-parallel.  Every rank must make the call with the same batch."""
    # Due to its mechanics, reinforce doesn't support testing (reinforce.py:80-81)
    learn = True
    policy = nets["policy_net"]
    vp = policy.__dict__.get("_recnn_vp")
    if vp is not None:
        critics = [nets.get(k) for k in ("value_net", "target_value_net", "target_policy_net")]
        if not _ids.is_item_ids(batch["action"]) or any(c is None or c.__dict__.get("_recnn_vp") is not vp
                                                        for c in critics):
            raise RuntimeError("reinforce_update feeds the policy's probabilities to its critic: a vocabulary-parallel "
                               "policy needs item-id batch actions and its critics, target policy included, sharded "
                               "with it (enable_vocab_parallel on the agent); on its own it trains through "
                               "ChooseREINFORCE only")
    dev = policy.linear1.weight.device
    if dev.type != "cuda":
        raise _lib.RecnnError("recnn_b200 update functions run on CUDA only (policy net is on %s); there is no CPU path" % dev)
    # item-id batch actions (an integer [N] tensor): the critic never sees a [N, num_items] matrix (_ids.py)
    ids = _ids.is_item_ids(batch["action"])
    if ids and not _ids._is_discrete(nets["target_policy_net"]):
        raise ValueError("item-id actions need a DiscreteActor target policy (nets['target_policy_net'])")
    state = batch["state"].to(dev)
    action = batch["action"].to(dev)

    predicted_probs = policy.select_action(state=state, action=action, K=params["K"], learn=learn, writer=writer, step=step)
    if not isinstance(writer, DummyWriter):
        writer.add_histogram("predicted_probs_std", predicted_probs.std(), step)
        writer.add_histogram("predicted_probs_mean", predicted_probs.mean(), step)
        mx = predicted_probs.max(dim=1).values
        writer.add_histogram("predicted_probs_max_mean", mx.mean(), step)
        writer.add_histogram("predicted_probs_max_std", mx.std(), step)
    if ids:
        reward = _ids.critic_value_of_probs(nets["value_net"], state, predicted_probs).detach()
    else:
        reward = nets["value_net"](state, predicted_probs).detach()
    policy.rewards.append(reward.mean())

    value_loss = value_update(batch, params, nets, optimizer, writer=writer, device=dev, debug=debug, learn=True, step=step)

    if step % params["policy_step"] == 0 and step > 0:
        policy_loss = params["reinforce"](policy, optimizer["policy_optimizer"])
        utils.soft_update(nets["value_net"], nets["target_value_net"], soft_tau=params["soft_tau"])
        utils.soft_update(nets["policy_net"], nets["target_policy_net"], soft_tau=params["soft_tau"])
        losses = {"value": value_loss.item(), "policy": policy_loss.item(), "step": step}
        utils.write_losses(writer, losses, kind="train" if learn else "test")
        return losses
