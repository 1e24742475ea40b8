"""recnn.data.utils equivalents for the FrameEnv minibatch path
(recnn/data/utils.py:7-10, :51-81, :161-187, :203-214, :265-276)."""
from __future__ import annotations

import numpy as np
import torch

from .. import _lib


def rolling_window(a, window):
    """All length-``window`` sliding windows of a 1-D array (utils.py:7-10), zero-copy."""
    return np.lib.stride_tricks.sliding_window_view(a, window)


def get_irsu(batch):
    return batch["items"], batch["ratings"], batch["sizes"], batch["users"]


def batch_tensor_embeddings(batch, item_embeddings_tensor, frame_size, *args, **kwargs):
    """Embed batch: continuous state, continuous action (utils.py:51-81), on the device.

    ``item_embeddings_tensor`` must live on a CUDA device (the table stays resident in HBM;
    only the int64 ids / fp32 ratings of the minibatch cross PCIe).  Returns the reference's
    dict (state, action, reward, next_state, done, meta) with CUDA tensors; bit-identical to
    the reference's CPU result."""
    items_t, ratings_t, sizes_t, users_t = get_irsu(batch)
    table = item_embeddings_tensor
    if table.device.type != "cuda":
        raise _lib.RecnnError("batch_tensor_embeddings: the embedding table must be on a CUDA device "
                              "(move it once with .cuda(); there is no CPU gather here)")
    if table.dtype != torch.float32 or not table.is_contiguous():
        raise ValueError("embedding table must be contiguous fp32")
    dev = table.device
    items = items_t.to(device=dev, dtype=torch.int64, non_blocking=True).contiguous()
    ratings = ratings_t.to(device=dev, dtype=torch.float32, non_blocking=True).contiguous()
    sizes = torch.as_tensor(sizes_t).to(device=dev, dtype=torch.int64, non_blocking=True).contiguous()
    n, f1 = ratings.shape
    if f1 != frame_size + 1 or tuple(items.shape) != (n, f1):
        raise ValueError("items/ratings must be [N, frame_size+1]")
    dim = table.shape[1]
    s_dim = frame_size * dim + frame_size
    state = torch.empty(n, s_dim, device=dev)
    next_state = torch.empty(n, s_dim, device=dev)
    action = torch.empty(n, dim, device=dev)
    reward = torch.empty(n, device=dev)
    done = torch.empty(n, device=dev)
    oob = torch.zeros(1, dtype=torch.int32, device=dev)
    with torch.cuda.device(dev):
        st = _lib.stream_ptr(dev)
        L = _lib.lib()
        _lib.check(L.recnn_frame_gather(table.data_ptr(), table.shape[0], dim, items.data_ptr(), ratings.data_ptr(),
                                        n, frame_size, state.data_ptr(), next_state.data_ptr(), action.data_ptr(),
                                        reward.data_ptr(), oob.data_ptr(), st))
        _lib.check(L.recnn_done_from_sizes(sizes.data_ptr(), sizes.numel(), frame_size, done.data_ptr(), n, st))
    if kwargs.get("check_bounds", True) and int(oob.item()) != 0:
        raise IndexError("item index out of range for the embedding table")   # torch indexing raises too
    return {"state": state, "action": action, "reward": reward, "next_state": next_state, "done": done,
            "meta": {"users": users_t, "sizes": sizes_t}}


def batch_contstate_discaction(batch, item_embeddings_tensor, frame_size, num_items, *args, one_hot=True, **kwargs):
    """Embed batch: continuous state, discrete action (utils.py:84-120), on the device.

    Same gather kernel as ``batch_tensor_embeddings`` for state / next_state / reward / done; the action is the item id
    of the last frame position -- returned as the reference's dense one-hot ``action`` [N, num_items] (what its
    ``Critic(1290, num_items, ...)`` consumes) and as ``action_index`` int64 [N].  ``one_hot=False`` returns the ids as
    ``action`` too: value_update / reinforce_update then run the critic without any [N, num_items] matrix."""
    out = batch_tensor_embeddings(batch, item_embeddings_tensor, frame_size, *args, **kwargs)
    dev = out["state"].device
    index = batch["items"][:, -1].to(device=dev, dtype=torch.int64)
    if int(index.max().item()) >= num_items or int(index.min().item()) < 0:
        raise RuntimeError("index out of range for a one-hot action of %d items" % num_items)   # scatter_ raises too
    if one_hot:
        dense = torch.zeros(index.shape[0], num_items, device=dev)
        dense.scatter_(1, index.view(-1, 1), 1)
        out["action"] = dense
    else:
        out["action"] = index
    out["action_index"] = index
    return out


def batch_frames(batch, item_embeddings_tensor, frame_size, *args, **kwargs):
    """embed_batch variant that does NOT materialise the state: returns the frame form
    (items, ratings, sizes, table) that ddpg_update / td3_update gather on the device
    inside the step.  Safe to run in a DataLoader worker (touches no CUDA memory)."""
    items_t, ratings_t, sizes_t, users_t = get_irsu(batch)
    return {"items": items_t, "ratings": ratings_t, "sizes": sizes_t, "users": users_t,
            "table": item_embeddings_tensor if item_embeddings_tensor.device.type == "cuda" else None,
            "meta": {"users": users_t, "sizes": sizes_t}}


def prepare_batch_static_size(batch, item_embeddings_tensor, frame_size=10, embed_batch=batch_tensor_embeddings):
    """DataLoader collate_fn (utils.py:161-187): per-user sliding windows of length
    frame_size+1, concatenated over the users of the batch, then ``embed_batch``."""
    items = np.concatenate([rolling_window(np.asarray(u["items"]), frame_size + 1) for u in batch], 0)
    rates = np.concatenate([rolling_window(np.asarray(u["rates"]), frame_size + 1) for u in batch], 0)
    out = {"items": torch.tensor(items), "users": torch.tensor([u["users"] for u in batch]),
           "ratings": torch.tensor(rates).float(), "sizes": torch.tensor([u["sizes"] for u in batch])}
    return embed_batch(batch=out, item_embeddings_tensor=item_embeddings_tensor, frame_size=frame_size)


def make_items_tensor(items_embeddings_key_dict):
    """dict {item key: embedding} -> dense table + key<->row maps (utils.py:203-214)."""
    keys = sorted(items_embeddings_key_dict.keys())
    key_to_id = {k: i for i, k in enumerate(keys)}
    id_to_key = {i: k for i, k in enumerate(keys)}
    table = torch.stack([torch.as_tensor(items_embeddings_key_dict[k]) for k in keys])
    return table, key_to_id, id_to_key


def get_base_batch(batch, device=torch.device("cuda"), done=True):
    """[state, action, reward[N,1], next_state, done[N,1]] on ``device`` (utils.py:265-276)."""
    b = [batch["state"], batch["action"], batch["reward"].unsqueeze(1), batch["next_state"]]
    if done:
        b.append(batch["done"].unsqueeze(1))
    else:
        b.append(torch.zeros_like(batch["reward"]).unsqueeze(1))   # the reference's branch is broken (:275)
    return [i.to(device) for i in b]
