"""The native calls of WorldModelEnv.predict_next_obs / predict_rew_end as torch custom ops (namespace `diamond_b200`).

The reference trainer wraps both methods in `torch.compile(..., mode="reduce-overhead")` when `training.compile_wm` is on
(trainer.py:182-184).  Dynamo cannot trace a ctypes call, so each native call is a custom op: Dynamo records it as one node
from its fake kernel, both methods compile without graph breaks, and the cudagraphs backend records the native kernels into
its graphs.  Eager calls go through the same ops and make the same C calls.

* The executor is reached through an int key (`key_of`), so no Python object appears in an op's schema.
* The module's state tensors are op inputs: cudagraph trees treat them as static inputs and re-record a graph when one is
  replaced.  A replay runs no Python, so the host-side re-pack check of NativeStateMixin does not run; the C entry points
  enqueue the fp16 weight packs inside the captured work instead, and every replay packs the parameters as they are then.
* The workspace is an op input as well: a recorded graph writes it in place, and a graph is re-recorded when it moves."""
import itertools
import weakref
from typing import List, Optional, Tuple

import torch
from torch import Tensor

_objects: "weakref.WeakValueDictionary[int, object]" = weakref.WeakValueDictionary()
_keys = itertools.count(1)


def key_of(obj) -> int:
    """The int key the ops reach `obj` (a DiffusionSampler or a RewEndModel) through.  Given out on first eager use; a
    compiled caller reads the attribute, so the key must exist before tracing (WorldModelEnv.reset makes sure of that)."""
    key = getattr(obj, "_op_key", None)
    if key is None:
        key = next(_keys)
        _objects[key] = obj
        obj.__dict__["_op_key"] = key
    return key


def _lookup(key: int):
    obj = _objects.get(key)
    if obj is None:
        raise RuntimeError(f"diamond_b200: no live executor has op key {key}")
    return obj


def mark_static(*tensors: Optional[Tensor]) -> None:
    """Persistent buffers a compiled caller reads or writes in place: cudagraphs use them at their address instead of copying
    them into the graph's own inputs, and accept in-place writes to them."""
    from torch._dynamo import mark_static_address

    for t in tensors:
        if t is not None:
            mark_static_address(t)


@torch.library.custom_op("diamond_b200::sample_ring", mutates_args=("frames", "traj", "workspace"))
def sample_ring(key: int, frames: Tensor, acts: Tensor, head: int, traj: Tensor, eps: Optional[Tensor], workspace: Tensor,
                params: List[Tensor]) -> None:
    """dmd_sampler_sample on a WorldModelEnv ring: frames (T, B, C, H, W) and acts (T, B) with logical slot k at physical
    slot (head + k) % T; the denoising trajectory goes to traj (num_sigmas, B, C, H, W) and the new frame to frames[head]."""
    _lookup(key)._sample_native(frames, acts, head, traj, eps, frames[head], workspace)


@sample_ring.register_fake
def _(key, frames, acts, head, traj, eps, workspace, params):
    return None


@torch.library.custom_op("diamond_b200::rew_end_predict", mutates_args=("workspace",))
def rew_end_predict(key: int, obs: Tensor, act: Tensor, next_obs: Tensor, hx: Optional[Tensor], cx: Optional[Tensor],
                    workspace: Tensor, params: List[Tensor]) -> Tuple[Tensor, Tensor, Tensor, Tensor]:
    """dmd_rew_end_predict: obs / next_obs (b, t, C, S, S) fp32, act (b, t) int64, hx / cx (b, lstm_dim) or None (zeros).
    Returns logits_rew (b, t, 3), logits_end (b, t, 2), hx and cx (b, lstm_dim), all new tensors."""
    return _lookup(key)._predict_native(obs, act, next_obs, hx, cx, workspace)


@rew_end_predict.register_fake
def _(key, obs, act, next_obs, hx, cx, workspace, params):
    b, t = obs.shape[:2]
    d = _lookup(key).cfg.lstm_dim
    return obs.new_empty(b, t, 3), obs.new_empty(b, t, 2), obs.new_empty(b, d), obs.new_empty(b, d)
